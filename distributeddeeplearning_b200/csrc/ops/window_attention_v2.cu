// Scaled-cosine shifted-window multi-head self-attention of Swin Transformer V2: window 8 (L = 64 tokens), head dim 32,
// the continuous position bias table T [225][heads] fp32 (16 sigmoid(cpb MLP), swin_v2.cu), a clamped per-head logit
// scale and the shifted-window mask, on the image-order qkv rows of the block, with padded maps handled natively.
//
// Layout (no pad, roll, partition, reverse or crop anywhere): qkv is the bf16 [N*H*W][3C] output of the qkv GEMM on the
// NHWC rows in image order; head h's Q, K and V are the 32 columns at 32h, C + 32h and 2C + 32h.  Windows tile the padded
// frame pH = ceil(H/8) 8, pW = ceil(W/8) 8: token i = (iy, ix) of window (wy, wx) of image n sits at
// y = (8 wy + iy + sy) mod pH, x = (8 wx + ix + sx) mod pW (torchvision's pad, roll by -shift and partition).  A token with
// y < H and x < W is real: it is read from row (n, y, x) and O goes back to that row of o [N*H*W][C].  The others are
// virtual and never touch qkv or o: torchvision pads the block input and its qkv linear runs with the k-bias zeroed, so a
// padded token has q = b_q, k = 0 and v = b_v (`qb` / `vb`, fp32 [C], null for zero).  lse [N*H*W][heads] fp32 is the
// natural-log log-sum-exp of the logits of every real (token, head).
//
// Logits: S_ij = (q_i . k_j) rq_i rk_j s_h + T[(iy - jy + 7) * 15 + (ix - jx + 7)][h] + M_ij with rq = 1 / max(|q|, 1e-12)
// (F.normalize), s_h = exp(min(logit_scale_h, ln 100)) and M_ij = -100 when i and j lie in different regions of the rolled
// padded frame: band(y') = 0 if y' < pH - 8, 1 if y' < pH - sy, else 2 (same for x), region = 3 band_y + band_x.  The
// norms are taken in fp32 from the bf16 tile and applied to the fp32 accumulator of the raw bf16 q . k: q-hat and k-hat
// are never rounded to bf16 (s_h would scale that rounding by up to 100x).
//
// Mapping: as window_attention.cu (window 7), one CTA of 4 warps per (window, head, image) in the forward, 16 query rows
// per warp on mma.sync.m16n8k16 bf16 with fp32 accumulators; L = 64 fills the 64-row tile, so no row is wasted and no
// key is masked to -inf.
//
// Backward: one CTA of 4 warps per (window row wy, head, image) walks wx = 0, 1, ... in order.  With dS = P o (dP - D):
//   dq_i = s_h rq_i (G_i - f_i (rq_i q_i . G_i) rq_i q_i),  G = (dS o rk^T) K           (dS column-scaled, registers)
//   dk_j = s_h rk_j (G'_j - f_j (rk_j k_j . G'_j) rk_j k_j),  G' = (rq o dS)^T Q          (dS row-scaled, shared bf16)
// where f = 1 when |q| >= 1e-12 (F.normalize's eps branch has no projection term); q . G = sum_j dS_ij c_ij / rq_i with
// c the cosine, so the projection needs no extra reduction.  dV = P^T dO.  Per CTA and head, in fixed orders, it keeps
// the sums of dS over the pairs of each of the 225 relative indices (masked pairs included), of dS o c (for the logit
// scale), of dq over the window's real tokens (q-bias) and of dv over all 64 tokens, virtual ones included (v-bias):
// the bias gradient of a qkv that carries [b_q, 0, b_v] on every token.  With bias_pad_only the two sums cover the
// virtual tokens only (their dq is 0): the gradient of b_q / b_v as the padding fill alone, for a qkv whose real rows
// are given.
// They go to part [N * nWy][heads][290]; a second kernel adds fixed chunks of (n, wy) and a third adds the chunks in
// order: dT [225][heads] = (written), dlogit_scale[h] += s_h sum(dS o c) (0 where the clamp is active), dbias[32h + d]
// and dbias[2C + 32h + d] += the q / v sums.  The k-bias entries are never written.  No atomics: every output is
// bit-identical run to run.  Shared memory is dynamic (59 KB: the fp32 dS tile of the table gradient alone is 18 KB).
#include <math.h>

#include "../common.cuh"
#include "ops.h"
#include "mma_tile.cuh"
#include "tc_utils.cuh"
#include "../launch.h"

namespace ddl {

namespace {

using namespace mma_tile;

constexpr int kWin = 8;
constexpr int kL = kWin * kWin;   // 64 tokens per window = the tile rows
constexpr int kD = 32;            // head dim
constexpr int kThreads = 128;     // 4 warps x 16 rows
constexpr int kLd = 40;           // shared row stride (bf16) of the Q / K / V / dO tiles
constexpr int kLdP = 72;          // shared row stride (bf16) of the P / dS tiles
constexpr int kLdF = 72;          // shared row stride (fp32) of the dS tile of the table gradient
constexpr int kTab = 225;         // (2 * 8 - 1)^2 relative positions
constexpr int kPer = kTab + 1 + 2 * kD;   // per (CTA, head): dT sums, sum dS o c, q-bias sums, v-bias sums
constexpr int kChunks = 64;       // first-level chunks of the parameter-gradient reduction
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn100 = 4.605170185988092f;
constexpr float kEps = 1e-12f;

struct WinArgs {
  const __nv_bfloat16* qkv;      // [N*H*W][3C]
  const __nv_bfloat16* o;        // [N*H*W][C]   (backward)
  const __nv_bfloat16* dout;     // [N*H*W][C]   (backward)
  const float* table;            // [225][heads]
  const float* scale;            // logit_scale [heads]
  const float* qb;               // q bias [C] of the virtual tokens (or null)
  const float* vb;               // v bias [C] of the virtual tokens (or null)
  __nv_bfloat16* out;            // forward: O; backward: dqkv
  float* lse;                    // [N*H*W][heads]
  float* part;                   // backward: [N * nWy][heads][kPer]
  int H, W, pH, pW, C, heads, sy, sx, nwy, nwx;
  int bias_pad_only;              // backward: the bias sums cover the virtual tokens only
};

struct BwdSmem {
  __nv_bfloat16 q[kL * kLd], k[kL * kLd], v[kL * kLd], dout[kL * kLd];
  __nv_bfloat16 p[kL * kLdP];    // P
  __nv_bfloat16 ds[kL * kLdP];   // rq_i dS_ij
  float dsf[kL * kLdF];          // dS (fp32) of every pair
  float d[kL], rq[kL], rk[kL], fq[kL], fk[kL];
  float bq[4][kD], bv[4][kD], dsc[4];
};

// image-order row of token i of window (wy, wx) of image n, or -1 for a virtual (padding) token
DDL_DEVICE long long token_row(const WinArgs& a, int n, int wy, int wx, int i) {
  int y = kWin * wy + (i >> 3) + a.sy, x = kWin * wx + (i & 7) + a.sx;
  if (y >= a.pH) y -= a.pH;
  if (x >= a.pW) x -= a.pW;
  if (y >= a.H || x >= a.W) return -1;
  return (static_cast<long long>(n) * a.H + y) * a.W + x;
}
// region of token i of window (wy, wx) in the rolled padded frame (0 when there is no shift)
DDL_DEVICE int token_region(const WinArgs& a, int wy, int wx, int i) {
  if ((a.sy | a.sx) == 0) return 0;
  const int y = kWin * wy + (i >> 3), x = kWin * wx + (i & 7);
  const int by = y < a.pH - kWin ? 0 : (y < a.pH - a.sy ? 1 : 2);
  const int bx = x < a.pW - kWin ? 0 : (x < a.pW - a.sx ? 1 : 2);
  return 3 * by + bx;
}
DDL_DEVICE int rel_key(int i) { return (i >> 3) * 15 + (i & 7); }

// T[rel(i, j)][h] + M_ij for query i (ri = rel_key(i) + 112, region gi) and key jj
DDL_DEVICE float bias_mask(const WinArgs& a, int h, int ri, int gi, int wy, int wx, int jj) {
  const float b = __ldg(a.table + (ri - rel_key(jj)) * a.heads + h);
  return token_region(a, wy, wx, jj) != gi ? b - 100.f : b;
}

// 64 rows x 32 bf16 of head columns `col` of the window's tokens into a tile of stride kLd: real tokens through
// cp.async, virtual ones set to bf16(fill[0..31]) (zero without a fill)
DDL_DEVICE void load_window(__nv_bfloat16* tile, const WinArgs& a, const __nv_bfloat16* base, int ld, int col,
                            const float* fill, int n, int wy, int wx, int tid) {
  const uint32_t t_s = tc::smem_u32(tile);
#pragma unroll
  for (int it = 0; it < (kL * 4) / kThreads; ++it) {
    const int c = tid + it * kThreads, r = c >> 2, ch = c & 3;
    const long long row = token_row(a, n, wy, wx, r);
    if (row >= 0) {
      tc::cp_async_16(t_s + static_cast<uint32_t>((r * kLd + ch * 8) * 2), base + row * ld + col + ch * 8, true);
    } else {
      uint4 v = make_uint4(0u, 0u, 0u, 0u);
      if (fill != nullptr) {
        const float* f = fill + ch * 8;
        v = make_uint4(pack_bf16x2(__ldg(f), __ldg(f + 1)), pack_bf16x2(__ldg(f + 2), __ldg(f + 3)),
                       pack_bf16x2(__ldg(f + 4), __ldg(f + 5)), pack_bf16x2(__ldg(f + 6), __ldg(f + 7)));
      }
      *reinterpret_cast<uint4*>(tile + r * kLd + ch * 8) = v;
    }
  }
}

// rq / rk = 1 / max(|row|, 1e-12) of the 64 Q rows (threads 0..63) and K rows (64..127) of the tiles; fq / fk (optional)
// = 1 where |row| >= 1e-12
DDL_DEVICE void inv_norms(const __nv_bfloat16* sQ, const __nv_bfloat16* sK, float* rq, float* rk, float* fq, float* fk,
                          int tid) {
  const int r = tid & (kL - 1);
  const __nv_bfloat16* row = (tid < kL ? sQ : sK) + r * kLd;
  float ss = 0.f;
#pragma unroll
  for (int c = 0; c < kD; c += 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + c);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = unpack_bf16x2(w[k]);
      ss = fmaf(f.x, f.x, fmaf(f.y, f.y, ss));
    }
  }
  const float nrm = sqrtf(ss);
  (tid < kL ? rq : rk)[r] = 1.f / fmaxf(nrm, kEps);
  if (fq != nullptr) (tid < kL ? fq : fk)[r] = nrm >= kEps ? 1.f : 0.f;
}

DDL_DEVICE float logit_scale(const WinArgs& a, int h) { return expf(fminf(__ldg(a.scale + h), kLn100)); }

__global__ void __launch_bounds__(kThreads) win2_attn_fwd_kernel(WinArgs a) {
  __shared__ __align__(128) __nv_bfloat16 sQ[kL * kLd];
  __shared__ __align__(128) __nv_bfloat16 sK[kL * kLd];
  __shared__ __align__(128) __nv_bfloat16 sV[kL * kLd];
  __shared__ float sRq[kL], sRk[kL];
  pdl_trigger();
  const int win = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int wy = win / a.nwx, wx = win - wy * a.nwx;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int ld = 3 * a.C;
  const uint32_t q_s = tc::smem_u32(sQ), k_s = tc::smem_u32(sK), v_s = tc::smem_u32(sV);
  pdl_wait();
  load_window(sQ, a, a.qkv, ld, h * kD, a.qb ? a.qb + h * kD : nullptr, n, wy, wx, tid);
  load_window(sK, a, a.qkv, ld, a.C + h * kD, nullptr, n, wy, wx, tid);
  load_window(sV, a, a.qkv, ld, 2 * a.C + h * kD, a.vb ? a.vb + h * kD : nullptr, n, wy, wx, tid);
  tc::cp_async_commit();
  tc::cp_async_wait<0>();
  __syncthreads();
  inv_norms(sQ, sK, sRq, sRk, nullptr, nullptr, tid);
  __syncthreads();
  const float sh = logit_scale(a, h);
  uint32_t qf[2][4];
#pragma unroll
  for (int kk = 0; kk < 2; ++kk) ldsm4(addr_a<kLd>(q_s, 16 * warp, 16 * kk, lane), qf[kk]);
  float s[8][4];
  mm_abt<kLd>(s, qf, k_s, lane);
  float m[2], l[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = 16 * warp + g + 8 * r;
    const int ri = rel_key(i) + 112, gi = token_region(a, wy, wx, i);
    const float qs = sRq[i] * sh;
    float mx = -INFINITY;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int jj = 8 * j + 2 * t + e;
        float& x = s[j][2 * r + e];
        x = fmaf(x, qs * sRk[jj], bias_mask(a, h, ri, gi, wy, wx, jj)) * kLog2e;
        mx = fmaxf(mx, x);
      }
    }
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
    const long long row = token_row(a, n, wy, wx, 16 * warp + g + 8 * r);
    if (row < 0) continue;
    const float inv = 1.f / l[r];
    __nv_bfloat16* dst = a.out + row * a.C + h * kD + 2 * t;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(acc[j][2 * r] * inv, acc[j][2 * r + 1] * inv);
    if (t == 0) a.lse[row * a.heads + h] = (m[r] + log2f(l[r])) * (1.f / kLog2e);
  }
}

// out = s rx (acc - f (rx x . acc) rx x) for the lane's two rows of a 16 x 32 accumulator tile whose rows are rows
// row0.. of the bf16 tile x (the normalisation gradient; the dot product over the 32 columns is reduced over the quad)
DDL_DEVICE void norm_grad(float (&acc)[4][4], const __nv_bfloat16* x, const float* rx, const float* fx, int row0,
                          float sh, int lane) {
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int i = row0 + g + 8 * r;
    float xv[8], dot = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(x + i * kLd + 8 * j + 2 * t));
      xv[2 * j] = f.x;
      xv[2 * j + 1] = f.y;
      dot = fmaf(f.x, acc[j][2 * r], fmaf(f.y, acc[j][2 * r + 1], dot));
    }
    dot += __shfl_xor_sync(0xffffffffu, dot, 1);
    dot += __shfl_xor_sync(0xffffffffu, dot, 2);
    const float ri = rx[i], pr = fx[i] * dot * ri * ri, sc = sh * ri;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      acc[j][2 * r] = sc * (acc[j][2 * r] - pr * xv[2 * j]);
      acc[j][2 * r + 1] = sc * (acc[j][2 * r + 1] - pr * xv[2 * j + 1]);
    }
  }
}

// column sums of a warp's 16 x 32 accumulator tile over the rows flagged in `use`, reduced over the 8 row groups of
// the warp in a fixed order; lanes 0..3 write columns 8j + 2t + e to dst[32]
DDL_DEVICE void col_sums(const float (&acc)[4][4], const bool (&use)[2], float* dst, int lane) {
  const int t = lane & 3;
  float c[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float v = (use[0] ? acc[j][e] : 0.f) + (use[1] ? acc[j][2 + e] : 0.f);
      v += __shfl_xor_sync(0xffffffffu, v, 4);
      v += __shfl_xor_sync(0xffffffffu, v, 8);
      v += __shfl_xor_sync(0xffffffffu, v, 16);
      c[2 * j + e] = v;
    }
  }
  if (lane < 4) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      dst[8 * j + 2 * t] = c[2 * j];
      dst[8 * j + 2 * t + 1] = c[2 * j + 1];
    }
  }
}

__global__ void __launch_bounds__(kThreads) win2_attn_bwd_kernel(WinArgs a) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  BwdSmem& sm = *reinterpret_cast<BwdSmem*>(smem_raw);
  pdl_trigger();
  const int wy = blockIdx.x, h = blockIdx.y, n = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
  const int C = a.C, ld = 3 * C;
  const uint32_t q_s = tc::smem_u32(sm.q), k_s = tc::smem_u32(sm.k), v_s = tc::smem_u32(sm.v);
  const uint32_t o_s = tc::smem_u32(sm.dout), p_s = tc::smem_u32(sm.p), s_s = tc::smem_u32(sm.ds);
  const float* qfill = a.qb ? a.qb + h * kD : nullptr;
  const float* vfill = a.vb ? a.vb + h * kD : nullptr;
  float dt_sum = 0.f, dt_sum2 = 0.f;   // table-gradient sums of relative index tid (and tid + 128 < 225)
  float aux = 0.f;                     // thread 127: sum dS o c; threads 0..31 / 32..63: q / v bias column sums
  pdl_wait();
  const float sh = logit_scale(a, h);
  for (int wx = 0; wx < a.nwx; ++wx) {
    load_window(sm.q, a, a.qkv, ld, h * kD, qfill, n, wy, wx, tid);
    load_window(sm.k, a, a.qkv, ld, C + h * kD, nullptr, n, wy, wx, tid);
    load_window(sm.v, a, a.qkv, ld, 2 * C + h * kD, vfill, n, wy, wx, tid);
    load_window(sm.dout, a, a.dout, C, h * kD, nullptr, n, wy, wx, tid);     // virtual queries: dO = 0
    tc::cp_async_commit();
    {   // D = rowsum(dO o O): two threads per row, 16 columns each (0 for a virtual row)
      const int r = tid >> 1, c0 = h * kD + (tid & 1) * 16;
      const long long row = token_row(a, n, wy, wx, r);
      float d = 0.f;
      if (row >= 0) {
        const size_t off = static_cast<size_t>(row) * C + c0;
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
      if ((tid & 1) == 0) sm.d[r] = d;
    }
    tc::cp_async_wait<0>();
    __syncthreads();
    inv_norms(sm.q, sm.k, sm.rq, sm.rk, sm.fq, sm.fk, tid);
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
      mm_abt<kLd>(dp, df, v_s, lane);
      float dsc = 0.f;
      bool real[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int i = 16 * warp + g + 8 * r;
        const long long row = token_row(a, n, wy, wx, i);
        real[r] = row >= 0;
        const float lse2 = real[r] ? a.lse[row * a.heads + h] * kLog2e : 0.f;
        const float dr = sm.d[i], rq = sm.rq[i];
        const int ri = rel_key(i) + 112, gi = token_region(a, wy, wx, i);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int q = 2 * r + e, jj = 8 * j + 2 * t + e;
            const float c = p[j][q] * rq * sm.rk[jj];
            const float lg = fmaf(c, sh, bias_mask(a, h, ri, gi, wy, wx, jj)) * kLog2e;
            const float pv = real[r] ? exp2f(lg - lse2) : 0.f;
            const float ds = pv * (dp[j][q] - dr);
            dsc = fmaf(ds, c, dsc);
            p[j][q] = pv;
            dp[j][q] = ds;
            sm.dsf[i * kLdF + jj] = ds;
          }
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int off = i * kLdP + 8 * j + 2 * t;
          *reinterpret_cast<uint32_t*>(sm.p + off) = pack_bf16x2(p[j][2 * r], p[j][2 * r + 1]);
          *reinterpret_cast<uint32_t*>(sm.ds + off) = pack_bf16x2(dp[j][2 * r] * rq, dp[j][2 * r + 1] * rq);
        }
      }
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) dsc += __shfl_xor_sync(0xffffffffu, dsc, o);
      if (lane == 0) sm.dsc[warp] = dsc;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
#pragma unroll
        for (int q = 0; q < 4; ++q) dp[j][q] *= sm.rk[8 * j + 2 * t + (q & 1)];
      }
      float dq[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dq[j][0] = dq[j][1] = dq[j][2] = dq[j][3] = 0.f;
      mm_pb<kLd>(dq, dp, k_s, lane);                                 // G = (dS o rk) K
      norm_grad(dq, sm.q, sm.rq, sm.fq, 16 * warp, sh, lane);
      const bool qu[2] = {real[0] != (a.bias_pad_only != 0), real[1] != (a.bias_pad_only != 0)};
      col_sums(dq, qu, sm.bq[warp], lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        if (!real[r]) continue;
        __nv_bfloat16* dst = a.out + token_row(a, n, wy, wx, 16 * warp + g + 8 * r) * ld + h * kD + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j)
          *reinterpret_cast<uint32_t*>(dst + 8 * j) = pack_bf16x2(dq[j][2 * r], dq[j][2 * r + 1]);
      }
    }
    __syncthreads();
    {
      float dk[4][4], dv[4][4];
#pragma unroll
      for (int j = 0; j < 4; ++j) dk[j][0] = dk[j][1] = dk[j][2] = dk[j][3] = dv[j][0] = dv[j][1] = dv[j][2] = dv[j][3] = 0.f;
      mm_atb<kLdP, kLd>(dv, p_s, 16 * warp, o_s, lane);              // dV = P^T dO
      mm_atb<kLdP, kLd>(dk, s_s, 16 * warp, q_s, lane);              // G' = (rq o dS)^T Q
      norm_grad(dk, sm.k, sm.rk, sm.fk, 16 * warp, sh, lane);
      long long rows[2];
      bool vu[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        rows[r] = token_row(a, n, wy, wx, 16 * warp + g + 8 * r);
        vu[r] = a.bias_pad_only == 0 || rows[r] < 0;
      }
      col_sums(dv, vu, sm.bv[warp], lane);
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const long long row = rows[r];
        if (row < 0) continue;
        __nv_bfloat16* dst = a.out + row * ld + h * kD + 2 * t;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          *reinterpret_cast<uint32_t*>(dst + C + 8 * j) = pack_bf16x2(dk[j][2 * r], dk[j][2 * r + 1]);
          *reinterpret_cast<uint32_t*>(dst + 2 * C + 8 * j) = pack_bf16x2(dv[j][2 * r], dv[j][2 * r + 1]);
        }
      }
    }
    if (tid < kTab) dt_sum += rel_sum<kWin, kLdF>(sm.dsf, tid);
    if (tid + kThreads < kTab) dt_sum2 += rel_sum<kWin, kLdF>(sm.dsf, tid + kThreads);
    if (tid == kThreads - 1) aux += ((sm.dsc[0] + sm.dsc[1]) + sm.dsc[2]) + sm.dsc[3];
    __syncthreads();                              // the tiles and sums are refilled by the next window
    if (tid < 2 * kD) {
      const float(*b)[kD] = tid < kD ? sm.bq : sm.bv;
      const int c = tid & (kD - 1);
      aux += ((b[0][c] + b[1][c]) + b[2][c]) + b[3][c];
    }
  }
  float* part = a.part + ((static_cast<size_t>(n) * a.nwy + wy) * a.heads + h) * kPer;
  part[tid] = dt_sum;
  if (tid + kThreads < kTab) part[tid + kThreads] = dt_sum2;
  if (tid == kThreads - 1) part[kTab] = aux;
  if (tid < 2 * kD) part[kTab + 1 + tid] = aux;
}

// second level: the chunks in order -> dtable[k][h] (written), dscale[h] += s_h sum(dS o c) unless clamped, dbias q / v
// slices += (each output optional)
__global__ void __launch_bounds__(kThreads) win2_grad_final_kernel(const float* __restrict__ chunk,
                                                                   const float* __restrict__ scale, float* dtable,
                                                                   float* dscale, float* dbias, int heads, int C) {
  pdl_trigger();
  pdl_wait();
  const int e = blockIdx.x * kThreads + threadIdx.x;
  if (e >= heads * kPer) return;
  float s = 0.f;
#pragma unroll 8
  for (int c = 0; c < kChunks; ++c) s += chunk[static_cast<size_t>(c) * heads * kPer + e];
  const int h = e / kPer, k = e - h * kPer;
  if (k < kTab) {
    if (dtable != nullptr) dtable[k * heads + h] = s;
  } else if (k == kTab) {
    const float ls = scale[h];
    if (dscale != nullptr) dscale[h] += ls <= kLn100 ? expf(ls) * s : 0.f;
  } else if (dbias != nullptr) {
    const int d = k - kTab - 1;                   // 0..31: q columns, 32..63: v columns
    dbias[(d < kD ? 0 : 2 * C - kD) + h * kD + d] += s;
  }
}

bool win_shape_ok(int N, int H, int W, int heads, int C, int sy, int sx) {
  if (!(N > 0 && N <= 65535 && heads > 0 && heads <= 65535 && C == kD * heads && H > 0 && W > 0)) return false;
  const int pH = (H + kWin - 1) / kWin * kWin, pW = (W + kWin - 1) / kWin * kWin;
  return static_cast<long long>(pH / kWin) * (pW / kWin) <= 2147483647LL && sy >= 0 &&
         sy < kWin && sx >= 0 && sx < kWin && (pH > kWin || sy == 0) && (pW > kWin || sx == 0);
}

WinArgs win_args(const __nv_bfloat16* qkv, const float* table, const float* scale, const float* qb, const float* vb,
                 int H, int W, int heads, int C, int sy, int sx) {
  WinArgs a{};
  a.qkv = qkv; a.table = table; a.scale = scale; a.qb = qb; a.vb = vb;
  a.H = H; a.W = W; a.C = C; a.heads = heads; a.sy = sy; a.sx = sx;
  a.pH = (H + kWin - 1) / kWin * kWin; a.pW = (W + kWin - 1) / kWin * kWin;
  a.nwy = a.pH / kWin; a.nwx = a.pW / kWin;
  return a;
}

}  // namespace

size_t window_attention_v2_bwd_scratch_floats(int N, int H, int heads) {
  return (static_cast<size_t>(N) * ((H + kWin - 1) / kWin) + kChunks) * heads * kPer;
}

cudaError_t launch_window_attention_v2_fwd(const __nv_bfloat16* qkv, const float* table, const float* scale,
                                           const float* qb, const float* vb, __nv_bfloat16* o, float* lse, int N, int H,
                                           int W, int heads, int C, int sy, int sx, cudaStream_t stream) {
  if (!win_shape_ok(N, H, W, heads, C, sy, sx)) return cudaErrorInvalidValue;
  WinArgs a = win_args(qkv, table, scale, qb, vb, H, W, heads, C, sy, sx);
  a.out = o; a.lse = lse;
  return launch_pdl(win2_attn_fwd_kernel, dim3(a.nwy * a.nwx, heads, N), dim3(kThreads), 0, stream, 1, a);
}

cudaError_t launch_window_attention_v2_bwd(const __nv_bfloat16* qkv, const float* table, const float* scale,
                                           const float* qb, const float* vb, const __nv_bfloat16* o,
                                           const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv,
                                           float* dtable, float* dscale, float* dbias, float* scratch, int N, int H,
                                           int W, int heads, int C, int sy, int sx, bool bias_pad_only,
                                           cudaStream_t stream) {
  if (!win_shape_ok(N, H, W, heads, C, sy, sx)) return cudaErrorInvalidValue;
  static const cudaError_t attr = cudaFuncSetAttribute(win2_attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                       static_cast<int>(sizeof(BwdSmem)));
  if (attr != cudaSuccess) return attr;
  WinArgs a = win_args(qkv, table, scale, qb, vb, H, W, heads, C, sy, sx);
  a.o = o; a.dout = dout; a.lse = const_cast<float*>(lse); a.out = dqkv; a.part = scratch;
  a.bias_pad_only = bias_pad_only ? 1 : 0;
  cudaError_t e = launch_pdl(win2_attn_bwd_kernel, dim3(a.nwy, heads, N), dim3(kThreads), sizeof(BwdSmem), stream, 1, a);
  if (e != cudaSuccess) return e;
  const int P = N * a.nwy, per = heads * kPer;
  float* chunk = scratch + static_cast<size_t>(P) * per;
  e = launch_pdl(grad_chunk_kernel<kThreads, kChunks>, dim3((per + kThreads - 1) / kThreads, kChunks), dim3(kThreads),
                 0, stream, 1, static_cast<const float*>(scratch), chunk, P, per);
  if (e != cudaSuccess) return e;
  return launch_pdl(win2_grad_final_kernel, dim3((per + kThreads - 1) / kThreads), dim3(kThreads), 0, stream, 1,
                    static_cast<const float*>(chunk), scale, dtable, dscale, dbias, heads, C);
}

}  // namespace ddl
