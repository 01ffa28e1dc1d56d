// Window attention of 49-token sequences, head dim 32, with a learned relative-position bias, on the image-order qkv rows
// of a block: the shifted-window multi-head self-attention of the Swin Transformer (V1), and the grid and window
// partition attention of MaxViT (torchvision's PartitionAttentionLayer).  One forward and one backward kernel template
// serve all three; a token-map type (ShiftedWindow, Partition<GRID>) gives the image row of every token, the sequence
// counts, the mask and the logit scale.
//
// Layout (no roll, partition, swap or reverse anywhere): qkv is the bf16 [N*H*W][3C] output of the qkv GEMM on the NHWC
// rows in image order; head h's Q, K and V are the 32 columns at 32h, C + 32h and 2C + 32h.  O of token t goes back to
// the same row of o [N*H*W][C] (proj's GEMM input as it is), which is the reverse partition.  lse [N*H*W][heads] fp32 is
// the natural-log log-sum-exp of the logits of every (token, head).  Token maps, token t = 7a + b of sequence (s0, s1)
// of image n:
//
//   Swin   window (wy, wx) of the map rolled by -(sy, sx): pixel ((7 wy + a + sy) mod H, (7 wx + b + sx) mod W), which is
//          torchvision's roll by -shift followed by the partition.
//   MaxViT grid (WindowPartition(p = H/7) + SwapAxes): pixel (a p + s0, b p + s1), the 49 tokens spaced p pixels apart.
//          window (WindowPartition(7)): pixel (7 s0 + a, 7 s1 + b).  Both cut a square H = W = 7p map (torchvision's
//          grid partition takes one p for both axes) into p x p sequences.
//
// Logits: S_tu = q_t . k_u * scale + table[(a - a' + 6) * 13 + (b - b' + 6)][h] + M_tu, with the fp32 parameter table
// [169][heads] read directly.  Swin's scale is the constant 1/sqrt(32); MaxViT's is an argument, because torchvision's
// RelativePositionalMultiHeadAttention scales k by feat_dim^-1/2, the layer's channel count C, not the head dim.  Only
// Swin has a mask: M = -100 when the shift is non-zero and t, u lie in different regions of the rolled frame: band(y') =
// 0 if y' < H - 7, 1 if y' < H - sy, else 2 (same for x), region = 3 band_y + band_x.  Both the index and the mask are
// computed from the token coordinates; no index or mask tensor is read.
//
// Mapping: one CTA of 4 warps per (sequence, head, image) in the forward; each warp owns 16 of the 64 query rows of the
// sequence tile (rows 49..63 are zero-filled and never stored) and runs mma.sync.m16n8k16 bf16 with fp32 accumulators
// (mma_tile.cuh).  Q, K and V come through cp.async into shared rows of 40 bf16 (80 B: 16-byte aligned, and the eight
// rows of an 8x8 ldmatrix fall in distinct banks).  The 16 x 64 score tile of a warp is one key block: keys 49..63 are
// -inf, the softmax is a single pass in fp32, base 2, scale folded in; P (the accumulators of n-tiles 2k, 2k+1) is the
// register A operand of O = P V.  Registers: Q fragment 8, scores 32, O accumulators 16.  Shared: 15 KB.
//
// Backward: one CTA of 4 warps per (sequence row s0, head, image) walks the sequences s1 = 0, 1, ... in order.  Per
// sequence it stages Q, K, V, dO (20 KB), forms D = rowsum(dO o O) from global memory, then per warp S,
// P = exp2(S' - lse'), dP = dO V^T, dS = P o (dP - D) and dQ = dS K * scale in registers; P and dS go to shared as bf16
// (stride 72, 18 KB) for the transposed products dV = P^T dO and dK = dS^T Q * scale of the warp's 16 key rows, and dS
// as fp32 (49 x 49, 9.4 KB) for the bias gradient: thread k < 169 adds the dS of every pair with relative index k, in a
// fixed order, to a running register sum over the CTA's sequences.  Masked pairs are included (the mask is a constant).
// The sums go to part [N * ny][heads][169] (ny sequence rows per image); a second kernel adds them over fixed chunks
// of (n, s0) and a third adds the chunks in order into dtable [169][heads].  No atomics anywhere: the results are bit-identical run to run.  dQ, dK
// and dV go into one bf16 [N*H*W][3C] buffer in qkv's layout.
#include <math.h>

#include "../common.cuh"
#include "ops.h"
#include "mma_tile.cuh"
#include "tc_utils.cuh"
#include "../launch.h"

namespace ddl {

namespace {

using namespace mma_tile;

constexpr int kWin = 7;
constexpr int kL = kWin * kWin;   // 49 tokens per sequence
constexpr int kD = 32;            // head dim
constexpr int kRows = 64;         // tile rows
constexpr int kThreads = 128;     // 4 warps x 16 rows
constexpr int kLd = 40;           // shared row stride (bf16) of the Q / K / V / dO tiles
constexpr int kLdP = 72;          // shared row stride (bf16) of the P / dS tiles
constexpr int kTab = 169;         // (2 * 7 - 1)^2 relative positions
constexpr int kChunks = 64;       // first-level chunks of the bias-gradient reduction
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kScale = 0.17677669529663687f;   // 1 / sqrt(32)

// Swin: window (s0, s1) = (wy, wx) of the map rolled by -(sy, sx), logits scaled by 1/sqrt(32), masked when shifted
struct ShiftedWindow {
  struct Args {
    const __nv_bfloat16* qkv;      // [N*H*W][3C]
    const __nv_bfloat16* o;        // [N*H*W][C]
    const __nv_bfloat16* dout;     // [N*H*W][C]   (backward)
    const float* table;            // [169][heads]
    __nv_bfloat16* out;            // forward: O; backward: dqkv
    float* lse;                    // [N*H*W][heads]
    float* part;                   // backward: [N * nWy][heads][169]
    int H, W, C, heads, sy, sx, nwy, nwx;
  };
  static constexpr bool kMasked = true;
  DDL_DEVICE static int ny(const Args& a) { return a.nwy; }   // sequence rows and columns per image
  DDL_DEVICE static int nx(const Args& a) { return a.nwx; }
  // by value: with a reference to the kernel argument here, nvcc schedules the forward differently from the literal
  DDL_DEVICE static float scale(Args) { return kScale; }
  DDL_DEVICE static size_t row(const Args& a, int n, int wy, int wx, int i) {
    const int iy = i / kWin, ix = i - iy * kWin;
    int y = kWin * wy + iy + a.sy, x = kWin * wx + ix + a.sx;
    if (y >= a.H) y -= a.H;
    if (x >= a.W) x -= a.W;
    return (static_cast<size_t>(n) * a.H + y) * a.W + x;
  }
  // region of token i in the rolled frame (0 when there is no shift)
  DDL_DEVICE static int region(const Args& a, int wy, int wx, int i) {
    if ((a.sy | a.sx) == 0) return 0;
    const int iy = i / kWin, ix = i - iy * kWin;
    const int y = kWin * wy + iy, x = kWin * wx + ix;
    const int by = y < a.H - kWin ? 0 : (y < a.H - a.sy ? 1 : 2);
    const int bx = x < a.W - kWin ? 0 : (x < a.W - a.sx ? 1 : 2);
    return 3 * by + bx;
  }
};

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

// MaxViT: sequence (s0, s1) of the grid (GRID) or window partition of a square map, logits scaled by the argument
template <bool GRID>
struct Partition {
  using Args = GridArgs;
  static constexpr bool kMasked = false;
  DDL_DEVICE static int ny(const Args& g) { return g.ns; }
  DDL_DEVICE static int nx(const Args& g) { return g.ns; }
  DDL_DEVICE static float scale(Args g) { return g.scale; }
  DDL_DEVICE static size_t row(const Args& g, int n, int i, int j, int t) {
    const int ta = t / kWin, tb = t - ta * kWin;
    const int y = GRID ? ta * g.ns + i : kWin * i + ta;
    const int x = GRID ? tb * g.ns + j : kWin * j + tb;
    return (static_cast<size_t>(n) * g.H + y) * g.H + x;
  }
};

DDL_DEVICE int rel_key(int i) { const int iy = i / kWin; return iy * 13 + (i - iy * kWin); }

// 64 rows x 32 bf16 of head columns `col` of the sequence's tokens (rows >= 49 zero-filled) into a tile of stride kLd
template <class Map>
DDL_DEVICE void load_seq(uint32_t tile, const typename Map::Args& a, const __nv_bfloat16* base, int ld, int col, int n,
                         int s0, int s1, int tid) {
#pragma unroll
  for (int it = 0; it < (kRows * 4) / kThreads; ++it) {
    const int c = tid + it * kThreads, r = c >> 2, ch = c & 3;
    const bool ok = r < kL;
    const __nv_bfloat16* src = base + (ok ? Map::row(a, n, s0, s1, r) : 0) * ld + col + ch * 8;
    tc::cp_async_16(tile + static_cast<uint32_t>((r * kLd + ch * 8) * 2), src, ok);
  }
}

// the base-2 logits of a warp's 16 x 64 score tile: s * scale + bias (+ mask), keys >= 49 at -inf
template <class Map>
DDL_DEVICE void logits(float (&s)[8][4], const typename Map::Args& a, int h, int s0, int s1, int row0, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = row0 + g + 8 * r;
    const int ii = i < kL ? i : 0;
    const int ri = rel_key(ii) + 84;
    int gi = 0;
    if constexpr (Map::kMasked) gi = Map::region(a, s0, s1, ii);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jj = 8 * j + 2 * t + e;
        float& x = s[j][2 * r + e];
        if (jj < kL) {
          float b = __ldg(a.table + (ri - rel_key(jj)) * a.heads + h);
          if constexpr (Map::kMasked) b += Map::region(a, s0, s1, jj) != gi ? -100.f : 0.f;
          x = fmaf(x, Map::scale(a), b) * kLog2e;
        } else {
          x = -INFINITY;
        }
      }
    }
  }
}

template <class Map>
__global__ void __launch_bounds__(kThreads) win_attn_fwd_kernel(typename Map::Args a) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[kRows * kLd];
  pdl_trigger();
  const int seq = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int s0 = seq / Map::nx(a), s1 = seq - s0 * Map::nx(a);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * a.C;
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV);
  pdl_wait();
  load_seq<Map>(q_s, a, a.qkv, ld, h * kD, n, s0, s1, tid);
  load_seq<Map>(k_s, a, a.qkv, ld, a.C + h * kD, n, s0, s1, tid);
  load_seq<Map>(v_s, a, a.qkv, ld, 2 * a.C + h * kD, n, s0, s1, tid);
  tc::cp_async_commit();
  tc::cp_async_wait<0>();
  __syncthreads();
  uint32_t qf[2][4];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) ldsm4(addr_a<kLd>(q_s, 16 * warp, 16 * kk, lane), qf[kk]);
  float s[8][4];
  mm_abt<kLd>(s, qf, k_s, lane);
  logits<Map>(s, a, h, s0, s1, 16 * warp, lane);
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
  mm_pb<kLd>(acc, s, v_s, lane);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = 16 * warp + g + 8 * r;
    if (i >= kL) continue;
    const size_t row = Map::row(a, n, s0, s1, i);
    const float inv = 1.f / l[r];
    __nv_bfloat16* dst = a.out + row * a.C + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) a.lse[row * a.heads + h] = (m[r] + log2f(l[r])) * (1.f / kLog2e);
  }
}

template <class Map>
__global__ void __launch_bounds__(kThreads) win_attn_bwd_kernel(typename Map::Args a) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[kRows * kLd];
  __shared__ __align__(128) __nv_bfloat16 sO[kRows * kLd];        // dO
  __shared__ __align__(128) __nv_bfloat16 sP[kRows * kLdP];
  __shared__ __align__(128) __nv_bfloat16 sS[kRows * kLdP];       // dS
  __shared__ float sSf[kL * kL];                                  // dS (fp32) of the real pairs
  __shared__ float sD[kRows];
  pdl_trigger();
  const int s0 = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int C = a.C, ld = 3 * C;
  const float scale = Map::scale(a);
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV), o_s = tc::smem_u32(sO);
  const uint32_t p_s = tc::smem_u32(sP), s_s = tc::smem_u32(sS);
  float dt_sum = 0.f, dt_sum2 = 0.f;         // bias-gradient sums of relative index tid (and tid + 128 < 169)
  pdl_wait();
  for (int s1 = 0; s1 < Map::nx(a); ++s1) {
    load_seq<Map>(q_s, a, a.qkv, ld, h * kD, n, s0, s1, tid);
    load_seq<Map>(k_s, a, a.qkv, ld, C + h * kD, n, s0, s1, tid);
    load_seq<Map>(v_s, a, a.qkv, ld, 2 * C + h * kD, n, s0, s1, tid);
    load_seq<Map>(o_s, a, a.dout, C, h * kD, n, s0, s1, tid);
    tc::cp_async_commit();
    {   // D = rowsum(dO o O): two threads per row, 16 columns each
      const int r = tid >> 1, c0 = h * kD + (tid & 1) * 16;
      float d = 0.f;
      if (r < kL) {
        const size_t off = Map::row(a, n, s0, s1, r) * C + c0;
#pragma unroll
        for (int v = 0; v < 2; ++v) {
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
      mm_abt<kLd>(p, qf, k_s, lane);
      logits<Map>(p, a, h, s0, s1, 16 * warp, lane);
      mm_abt<kLd>(dp, df, v_s, lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = 16 * warp + g + 8 * r;
        const bool ok = i < kL;
        const float lse2 = ok ? a.lse[Map::row(a, n, s0, s1, i) * a.heads + h] * kLog2e : 0.f;
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
          const int off = (16 * warp + g + 8 * r) * kLdP + 8 * j + 2 * t;
          *reinterpret_cast<uint32_t*>(sP + off) = pack_bf16x2(p[j][2 * r], p[j][2 * r + 1]);
          *reinterpret_cast<uint32_t*>(sS + off) = pack_bf16x2(dp[j][2 * r], dp[j][2 * r + 1]);
        }
      }
      float dq[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;
      mm_pb<kLd>(dq, dp, k_s, lane);                                 // dQ = dS K
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = 16 * warp + g + 8 * r;
        if (i >= kL) continue;
        __nv_bfloat16* dst = a.out + Map::row(a, n, s0, s1, i) * ld + h * kD + 2 * t;
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
      mm_atb<kLdP, kLd>(dv, p_s, 16 * warp, o_s, lane);              // dV = P^T dO
      mm_atb<kLdP, kLd>(dk, s_s, 16 * warp, q_s, lane);              // dK = dS^T Q
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int k = 16 * warp + g + 8 * r;
        if (k >= kL) continue;
        __nv_bfloat16* dst = a.out + Map::row(a, n, s0, s1, k) * ld + h * kD + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          *reinterpret_cast<uint32_t*>(dst + C + 8 * j) = pack_bf16x2(dk[j][2 * r] * scale, dk[j][2 * r + 1] * scale);
          *reinterpret_cast<uint32_t*>(dst + 2 * C + 8 * j) = pack_bf16x2(dv[j][2 * r], dv[j][2 * r + 1]);
        }
      }
    }
    // bias gradient: the pairs (i, j) with iy - jy = dy and ix - jx = dx, in row-major order of i
    if (tid < kTab) dt_sum += rel_sum<kWin, kL>(sSf, tid);
    if (tid + kThreads < kTab) dt_sum2 += rel_sum<kWin, kL>(sSf, tid + kThreads);
    __syncthreads();                              // the tiles and sSf are refilled by the next sequence
  }
  float* part = a.part + ((static_cast<size_t>(n) * Map::ny(a) + s0) * a.heads + h) * kTab;
  if (tid < kTab) part[tid] = dt_sum;
  if (tid + kThreads < kTab) part[tid + kThreads] = dt_sum2;
}

// second level: dtable[k][h] += sum over the chunks in order
__global__ void __launch_bounds__(kThreads) win_bias_grad_final_kernel(const float* __restrict__ chunk,
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

// the bias gradient from the P = N * rows partial sums at the start of scratch: chunks after them, then dtable
cudaError_t launch_bias_grad(float* scratch, float* dtable, int P, int heads, cudaStream_t stream) {
  const int per = heads * kTab;
  float* chunk = scratch + static_cast<size_t>(P) * per;
  cudaError_t e = launch_pdl(grad_chunk_kernel<kThreads, kChunks>, dim3((per + kThreads - 1) / kThreads, kChunks),
                             dim3(kThreads), 0, stream, 1, static_cast<const float*>(scratch), chunk, P, per);
  if (e != cudaSuccess) return e;
  return launch_pdl(win_bias_grad_final_kernel, dim3((per + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(chunk), dtable, heads);
}

bool win_shape_ok(int N, int H, int W, int heads, int C, int sy, int sx) {
  return N > 0 && N <= 65535 && heads > 0 && heads <= 65535 && C == kD * heads && H > 0 && W > 0 &&
         H % kWin == 0 && W % kWin == 0 && (H / kWin) * (W / kWin) <= 65535 && sy >= 0 && sy < kWin && sx >= 0 &&
         sx < kWin && (H > kWin || sy == 0) && (W > kWin || sx == 0);
}

ShiftedWindow::Args win_args(const __nv_bfloat16* qkv, int H, int W, int heads, int C, int sy, int sx) {
  ShiftedWindow::Args a{};
  a.qkv = qkv; a.H = H; a.W = W; a.C = C; a.heads = heads; a.sy = sy; a.sx = sx;
  a.nwy = H / kWin; a.nwx = W / kWin;
  return a;
}

bool grid_shape_ok(int N, int H, int W, int heads, int C) {
  return N > 0 && N <= 65535 && heads > 0 && heads <= 65535 && C == kD * heads && H > 0 && H == W && H % kWin == 0 &&
         (H / kWin) * (H / kWin) <= 65535;
}

GridArgs grid_args(const __nv_bfloat16* qkv, int H, int heads, int C, float scale) {
  GridArgs g{};
  g.qkv = qkv; g.H = H; g.C = C; g.heads = heads; g.ns = H / kWin; g.scale = scale;
  return g;
}

}  // namespace

size_t window_attention_bwd_scratch_floats(int N, int H, int heads) {
  return (static_cast<size_t>(N) * (H / kWin) + kChunks) * heads * kTab;
}

// the same partial-sum and chunk layout: N * (H / 7) sequence rows
size_t grid_attention_bwd_scratch_floats(int N, int H, int heads) {
  return window_attention_bwd_scratch_floats(N, H, heads);
}

cudaError_t launch_window_attention_fwd(const __nv_bfloat16* qkv, const float* table, __nv_bfloat16* o, float* lse,
                                        int N, int H, int W, int heads, int C, int sy, int sx, cudaStream_t stream) {
  if (!win_shape_ok(N, H, W, heads, C, sy, sx)) return cudaErrorInvalidValue;
  ShiftedWindow::Args a = win_args(qkv, H, W, heads, C, sy, sx);
  a.table = table; a.out = o; a.lse = lse;
  const dim3 grid(a.nwy * a.nwx, heads, N);
  return launch_pdl(win_attn_fwd_kernel<ShiftedWindow>, grid, dim3(kThreads), 0, stream, 1, a);
}

cudaError_t launch_window_attention_bwd(const __nv_bfloat16* qkv, const float* table, const __nv_bfloat16* o,
                                        const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv, float* dtable,
                                        float* scratch, int N, int H, int W, int heads, int C, int sy, int sx,
                                        cudaStream_t stream) {
  if (!win_shape_ok(N, H, W, heads, C, sy, sx)) return cudaErrorInvalidValue;
  ShiftedWindow::Args a = win_args(qkv, H, W, heads, C, sy, sx);
  a.table = table; a.o = o; a.dout = dout; a.lse = const_cast<float*>(lse); a.out = dqkv; a.part = scratch;
  const cudaError_t e = launch_pdl(win_attn_bwd_kernel<ShiftedWindow>, dim3(a.nwy, heads, N), dim3(kThreads), 0,
                                   stream, 1, a);
  return e != cudaSuccess ? e : launch_bias_grad(scratch, dtable, N * a.nwy, heads, stream);
}

cudaError_t launch_grid_attention_fwd(const __nv_bfloat16* qkv, const float* table, __nv_bfloat16* o, float* lse,
                                      int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream) {
  if (!grid_shape_ok(N, H, W, heads, C)) return cudaErrorInvalidValue;
  GridArgs g = grid_args(qkv, H, heads, C, scale);
  g.table = table; g.out = o; g.lse = lse;
  const dim3 blocks(g.ns * g.ns, heads, N);
  return grid ? launch_pdl(win_attn_fwd_kernel<Partition<true>>, blocks, dim3(kThreads), 0, stream, 1, g)
              : launch_pdl(win_attn_fwd_kernel<Partition<false>>, blocks, dim3(kThreads), 0, stream, 1, g);
}

cudaError_t launch_grid_attention_bwd(const __nv_bfloat16* qkv, const float* table, const __nv_bfloat16* o,
                                      const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv, float* dtable,
                                      float* scratch, int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream) {
  if (!grid_shape_ok(N, H, W, heads, C)) return cudaErrorInvalidValue;
  GridArgs g = grid_args(qkv, H, heads, C, scale);
  g.table = table; g.o = o; g.dout = dout; g.lse = const_cast<float*>(lse); g.out = dqkv; g.part = scratch;
  const dim3 blocks(g.ns, heads, N), threads(kThreads);
  const cudaError_t e = grid ? launch_pdl(win_attn_bwd_kernel<Partition<true>>, blocks, threads, 0, stream, 1, g)
                             : launch_pdl(win_attn_bwd_kernel<Partition<false>>, blocks, threads, 0, stream, 1, g);
  return e != cudaSuccess ? e : launch_bias_grad(scratch, dtable, N * g.ns, heads, stream);
}

}  // namespace ddl
