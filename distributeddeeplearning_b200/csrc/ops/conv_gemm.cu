// wgmma / TMA implicit-GEMM convolution kernels for sm_90a (bf16 in, fp32 accumulate).
//
// Replaces the cuDNN conv fwd / bwd-data / bwd-filter and cuBLAS FC calls of the reference's
// training step (SURVEY.md K2, K3, K4, K10; N4, N5).  All three passes are GEMMs on NHWC data:
//
//   fwd    Y[m][co]  = sum_k  im2col(X)[m][k]  * W[co][k]          k = (r, s, ci)
//   dgrad  dX[m][ci] = sum_k  im2colT(dY)[m][k] * W[co][(r,s,ci)]   k = (r, s, co)   (B is MN-major)
//   wgrad  dW[co][k] = sum_m  dY[m][co]        * im2col(X)[m][k]    (A and B are MN-major, split-K)
//
// One CTA = 13 warps:
//   warps 0-7  two consumer warpgroups: warpgroup g issues the wgmma of accumulator rows [64g, 64g+64) of the
//              128-row tile and keeps them in registers, then runs the epilogue (registers -> smem staging ->
//              coalesced global stores; fused BN statistics / bias / ReLU / residual add)
//   warps 8-11 im2col producers in the gather modes (strided convs, stem): each thread owns one 128-byte row of the
//              operand tile and fills it with cp.async (zero-fill = padding / tails) in the 128B-swizzled image wgmma
//              reads; idle in the TMA-fed modes
//   warp 12    TMA producer: weights always; the activation operand too whenever it is a plain matrix
//              (2-D map) or a stride-1 convolution window (ONE 4-D box per filter tap — the hardware does
//              the im2col, out-of-bounds coordinates supply the zero padding)
// Stages are handed over with mbarriers (full/empty ring); a consumer warp releases a stage once the wgmma group that
// read it has retired.  The ring is as deep as shared memory allows (one CTA per SM).
#include "conv_gemm.cuh"
#include "tc_utils.cuh"
#include "../launch.h"

#include <dlfcn.h>

namespace ddl {

int g_pdl = 1;        // launch.h: opted-in kernels are launched with programmatic stream serialization

using namespace tc;

namespace {

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;                       // bf16 elements = 128 bytes = one swizzle row
constexpr int kATileBytes = kBlockM * 128;        // 16 KB
constexpr int kEpiThreads = 256;                  // warps 0-7: the two consumer warpgroups
constexpr int kProducerWarp0 = 8;                 // warps 8-11: cp.async gather producers
constexpr int kProducerThreads = 128;
constexpr int kTmaWarp = 12;
constexpr int kThreads = 13 * 32;
constexpr int kLag = 2;                           // cp.async groups kept in flight per producer
constexpr int kMaxStages = 8;

template <int BLOCK_N>
struct FwdCfg {
  static constexpr int kBTileBytes = BLOCK_N * 128;
  static constexpr int kStageBytes = kATileBytes + kBTileBytes;
  static constexpr int kPitch = BLOCK_N * 2 + 16;                 // epilogue staging row pitch (bytes)
  static constexpr int kEpiBytes = ((kBlockM * kPitch + 1023) / 1024) * 1024;
  static constexpr int kFixed = kEpiBytes + 256 /*barriers*/ + 8192 /*stats scratch*/ + 1024 /*alignment*/;
  static constexpr int kMaxStagesN = (232448 - kFixed) / kStageBytes > kMaxStages ? kMaxStages
                                                                                   : (232448 - kFixed) / kStageBytes;
  static constexpr int smem_bytes(int stages) { return stages * kStageBytes + kFixed; }
};

DDL_DEVICE void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" :: "r"(id), "r"(nthreads) : "memory");
}

DDL_DEVICE void tma_load_4d(uint32_t dst_smem, const CUtensorMap* m, int c0, int c1, int c2, int c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
      :: "r"(dst_smem), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}

DDL_DEVICE void tma_load_5d(uint32_t dst_smem, const CUtensorMap* m, int c0, int c1, int c2, int c3, int c4,
                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
      :: "r"(dst_smem), "l"(reinterpret_cast<uint64_t>(m)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4),
         "r"(smem_u32(bar))
      : "memory");
}

constexpr bool mode_a_tma(int mode) {
  return mode == kConvGemm || mode == kConvTileFwd || mode == kConvTileDgrad || mode == kConvGemmDgrad ||
         mode == kConvStemTma;
}
constexpr bool mode_b_mn(int mode) { return mode == kConvDgrad || mode == kConvTileDgrad || mode == kConvGemmDgrad; }
constexpr bool mode_tile(int mode) { return mode == kConvTileFwd || mode == kConvTileDgrad || mode == kConvStemTma; }
constexpr bool mode_stem(int mode) { return mode == kConvStem || mode == kConvStemTma; }


// ---------------------------------------------------------------------------------------------
// epilogue building blocks
// ---------------------------------------------------------------------------------------------
// All staging traffic uses 32-bit shared-window addresses (ld/st.shared): generic LD/ST through the aligned
// dynamic-smem pointer cost 64-bit address arithmetic per access.
DDL_DEVICE void sts128(uint32_t addr, uint32_t x, uint32_t y, uint32_t z, uint32_t w) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "r"(x), "r"(y), "r"(z), "r"(w) : "memory");
}
DDL_DEVICE uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
DDL_DEVICE void sts32(uint32_t addr, uint32_t v) { asm volatile("st.shared.b32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }
DDL_DEVICE uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
DDL_DEVICE float lds_f32(uint32_t addr) { return __uint_as_float(lds32(addr)); }

// Attribution experiments (tools/epi_probe.py): bits 12-14 of the variant word switch epilogue phases OFF.  The results
// are then wrong by construction; production launches never set them (native.py builds variant words from bits 0-8).
constexpr int kDbgNoStats = 1 << 12;   // no statistics pass (and no atomics)
constexpr int kDbgNoStore = 1 << 13;   // no global stores
constexpr int kDbgNoDrain = 1 << 14;   // no accumulator -> staging copy

// wgmma accumulator fragment of this thread -> (dequantise, bias, ReLU) -> bf16 -> staging rows r0 and r0 + 8.
// `z0` / `z1`: the row lies outside the image (tile modes) and is staged as zeros.
template <int BLOCK_N, bool BIAS_RELU>
DDL_DEVICE void epi_acc_to_stage(const float (&acc)[BLOCK_N / 2], uint32_t stg, int r0, bool z0, bool z1,
                                 const ConvArgs& a, int n0, float deq) {
  constexpr int kPitch = BLOCK_N * 2 + 16;
  if (a.variant & kDbgNoDrain) return;
  const uint32_t row0 = stg + r0 * kPitch, row1 = row0 + 8 * kPitch;
  const int cq = 2 * (threadIdx.x & 3);
#pragma unroll
  for (int j = 0; j < BLOCK_N / 8; ++j) {
    const int c = 8 * j + cq;
    float x0 = acc[4 * j] * deq, x1 = acc[4 * j + 1] * deq, y0 = acc[4 * j + 2] * deq, y1 = acc[4 * j + 3] * deq;
    if (BIAS_RELU) {
      if (a.bias) {
        const float b0 = (n0 + c < a.n_valid) ? a.bias[n0 + c] : 0.f;
        const float b1 = (n0 + c + 1 < a.n_valid) ? a.bias[n0 + c + 1] : 0.f;
        x0 += b0; x1 += b1; y0 += b0; y1 += b1;
      }
      if (a.relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
    }
    sts32(row0 + c * 2, z0 ? 0u : pack_bf16x2(x0, x1));
    sts32(row1 + c * 2, z1 ? 0u : pack_bf16x2(y0, y1));
  }
}

// ---- fp32 pairs (two statistics lanes per 64-bit register pair) -------------------------------------------------
DDL_DEVICE uint64_t f2_pack(float lo, float hi) {
  uint64_t d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(lo), "f"(hi));
  return d;
}
DDL_DEVICE void f2_unpack(uint64_t v, float& lo, float& hi) { asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v)); }
DDL_DEVICE uint64_t f2_from_bf16x2(uint32_t u) {            // {bf16 lo, bf16 hi} -> {fp32, fp32}: two ALU ops
  uint64_t d;
  const uint32_t lo = u << 16, hi = u & 0xffff0000u;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "r"(lo), "r"(hi));
  return d;
}
DDL_DEVICE uint64_t f2_add(uint64_t a, uint64_t b) {
  float a0, a1, b0, b1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  return f2_pack(a0 + b0, a1 + b1);
}
DDL_DEVICE uint64_t f2_fma(uint64_t a, uint64_t b, uint64_t c) {
  float a0, a1, b0, b1, c0, c1;
  f2_unpack(a, a0, a1);
  f2_unpack(b, b0, b1);
  f2_unpack(c, c0, c1);
  return f2_pack(fmaf(a0, b0, c0), fmaf(a1, b1, c1));
}

// Per-thread partial BN statistics of 8 consecutive output channels (4 pairs each), flushed with warp shuffles, one
// shared-memory fold and one atomic per channel and statistic.
struct StatAcc {
  uint64_t s[4], q[4];
  int n0;                       // first channel of the tile column these sums belong to; -1 = empty
  DDL_DEVICE void clear() {
#pragma unroll
    for (int i = 0; i < 4; ++i) { s[i] = 0ull; q[i] = 0ull; }
    n0 = -1;
  }
};

// Fold the staged bf16 tile (row pitch BLOCK_N*2+16) into `acc`.  Thread = (column group of 8, row slice); invalid rows
// hold zeros.  Entered by all kEpiThreads epilogue threads after the staging writes were made visible (named barrier 1).
template <int BLOCK_N, bool TILE>
DDL_DEVICE void epi_stats_accum(uint32_t stg, int etid, const ConvArgs& a, int n0, int m0, StatAcc& acc) {
  constexpr int kPitch = BLOCK_N * 2 + 16;
  constexpr int kColGroups = BLOCK_N / 8;                 // 16 (N=128) or 8 (N=64)
  constexpr int kSlices = kEpiThreads / kColGroups;       // row slices
  constexpr int kRowsPer = kBlockM / kSlices;             // rows per thread
  if (a.variant & kDbgNoStats) return;
  const int cg = etid % kColGroups;
  const int sl = etid / kColGroups;
  const uint32_t p0 = stg + (sl * kRowsPer) * kPitch + cg * 16;
  acc.n0 = n0;
  if (a.bnr_y == nullptr) {
#pragma unroll
    for (int r = 0; r < kRowsPer; ++r) {
      const uint4 u = lds128(p0 + r * kPitch);
      uint64_t f;
      f = f2_from_bf16x2(u.x); acc.s[0] = f2_add(acc.s[0], f); acc.q[0] = f2_fma(f, f, acc.q[0]);
      f = f2_from_bf16x2(u.y); acc.s[1] = f2_add(acc.s[1], f); acc.q[1] = f2_fma(f, f, acc.q[1]);
      f = f2_from_bf16x2(u.z); acc.s[2] = f2_add(acc.s[2], f); acc.q[2] = f2_fma(f, f, acc.q[2]);
      f = f2_from_bf16x2(u.w); acc.s[3] = f2_add(acc.s[3], f); acc.q[3] = f2_fma(f, f, acc.q[3]);
    }
    return;
  }
  // fused BN-backward reduction (see ConvArgs::bnr_y): S1 = sum dm, S2 = sum dm * y with the ReLU mask of the BN
  // recomputed from y.  The y tile is read with the same coalesced 16-byte accesses the stores use.
  const int c0 = n0 + cg * 8;
  if (c0 >= a.n_valid) return;
  uint64_t sc[4], sh[4];
#pragma unroll
  for (int qd = 0; qd < 2; ++qd) {
    const float4 g4 = reinterpret_cast<const float4*>(a.bnr_gamma + c0)[qd];
    const float4 b4 = reinterpret_cast<const float4*>(a.bnr_beta + c0)[qd];
    const float4 m4 = reinterpret_cast<const float4*>(a.bnr_mean + c0)[qd];
    const float4 i4 = reinterpret_cast<const float4*>(a.bnr_invstd + c0)[qd];
    const float s0 = g4.x * i4.x, s1 = g4.y * i4.y, s2 = g4.z * i4.z, s3 = g4.w * i4.w;
    sc[2 * qd] = f2_pack(s0, s1); sh[2 * qd] = f2_pack(b4.x - m4.x * s0, b4.y - m4.y * s1);
    sc[2 * qd + 1] = f2_pack(s2, s3); sh[2 * qd + 1] = f2_pack(b4.z - m4.z * s2, b4.w - m4.w * s3);
  }
#pragma unroll 2
  for (int r = 0; r < kRowsPer; ++r) {
    const int row = sl * kRowsPer + r;
    int m;
    if (TILE) m = static_cast<int>(lds32(stg + row * kPitch + BLOCK_N * 2));
    else m = (m0 + row) < a.M ? (m0 + row) : -1;
    if (m < 0) continue;
    const uint4 u = lds128(p0 + r * kPitch);
    const uint4 yv = *reinterpret_cast<const uint4*>(a.bnr_y + static_cast<size_t>(m) * a.ldc + c0);
    const uint32_t du[4] = {u.x, u.y, u.z, u.w}, yu[4] = {yv.x, yv.y, yv.z, yv.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint64_t y2 = f2_from_bf16x2(yu[j]);
      float z0, z1, d0, d1;
      f2_unpack(f2_fma(y2, sc[j], sh[j]), z0, z1);
      f2_unpack(f2_from_bf16x2(du[j]), d0, d1);
      const uint64_t dm = f2_pack(z0 > 0.f ? d0 : 0.f, z1 > 0.f ? d1 : 0.f);
      acc.s[j] = f2_add(acc.s[j], dm);
      acc.q[j] = f2_fma(dm, y2, acc.q[j]);
    }
  }
}

// Publish `acc` (sums of tile column acc.n0) and clear it.  Contains one named barrier: must be reached by all
// kEpiThreads epilogue threads together; `red` = [epi warps][2][BLOCK_N] floats of scratch.  A later flush may rewrite
// the scratch only after another barrier of the same group (every caller has one per tile / chunk in between).
template <int BLOCK_N>
DDL_DEVICE void epi_stats_flush(uint32_t red, int etid, int ew, const ConvArgs& a, StatAcc& acc) {
  constexpr int kColGroups = BLOCK_N / 8;
  if (a.variant & kDbgNoStats) { acc.clear(); return; }
  const int cg = etid % kColGroups;
  const int n0 = acc.n0;
  // threads with the same column group inside a warp: lanes cg, cg+kColGroups, ... -> xor shuffles
#pragma unroll
  for (int off = kColGroups; off < 32; off <<= 1) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      acc.s[i] = f2_add(acc.s[i], __shfl_xor_sync(0xffffffffu, acc.s[i], off));
      acc.q[i] = f2_add(acc.q[i], __shfl_xor_sync(0xffffffffu, acc.q[i], off));
    }
  }
  // cross-warp fold in shared memory ([epi warp][2][BLOCK_N] floats), then ONE atomic per channel and statistic
  if ((threadIdx.x & 31) < kColGroups) {
    const uint32_t rb = red + ((ew * 2) * BLOCK_N + cg * 8) * 4;
    sts128(rb, static_cast<uint32_t>(acc.s[0]), static_cast<uint32_t>(acc.s[0] >> 32), static_cast<uint32_t>(acc.s[1]),
           static_cast<uint32_t>(acc.s[1] >> 32));
    sts128(rb + 16, static_cast<uint32_t>(acc.s[2]), static_cast<uint32_t>(acc.s[2] >> 32),
           static_cast<uint32_t>(acc.s[3]), static_cast<uint32_t>(acc.s[3] >> 32));
    sts128(rb + BLOCK_N * 4, static_cast<uint32_t>(acc.q[0]), static_cast<uint32_t>(acc.q[0] >> 32),
           static_cast<uint32_t>(acc.q[1]), static_cast<uint32_t>(acc.q[1] >> 32));
    sts128(rb + BLOCK_N * 4 + 16, static_cast<uint32_t>(acc.q[2]), static_cast<uint32_t>(acc.q[2] >> 32),
           static_cast<uint32_t>(acc.q[3]), static_cast<uint32_t>(acc.q[3] >> 32));
  }
  acc.clear();
  named_bar_sync(1, kEpiThreads);
  if (a.bnr_y == nullptr) {
    for (int c = etid; c < 2 * BLOCK_N; c += kEpiThreads) {
      const int which = c / BLOCK_N, col = c - which * BLOCK_N;
      float v = 0.f;
#pragma unroll
      for (int wq = 0; wq < kEpiThreads / 32; ++wq) v += lds_f32(red + ((wq * 2 + which) * BLOCK_N + col) * 4);
      if (n0 + col < a.n_valid) atomicAdd((which ? a.sumsq : a.sum) + n0 + col, v);
    }
  } else {
    for (int col = etid; col < BLOCK_N; col += kEpiThreads) {      // dbeta += S1, dgamma += invstd * (S2 - mean * S1)
      float t1 = 0.f, t2 = 0.f;
#pragma unroll
      for (int wq = 0; wq < kEpiThreads / 32; ++wq) {
        t1 += lds_f32(red + ((wq * 2 + 0) * BLOCK_N + col) * 4);
        t2 += lds_f32(red + ((wq * 2 + 1) * BLOCK_N + col) * 4);
      }
      const int ch = n0 + col;
      if (ch < a.n_valid) {
        atomicAdd(a.sum + ch, t1);
        atomicAdd(a.sumsq + ch, a.bnr_invstd[ch] * (t2 - a.bnr_mean[ch] * t1));
      }
    }
  }
}

// The coalesced 16-byte global stores of the staged tile (optional `+= add`, optional zero-fill of the three stride-2
// siblings): thread = (16-byte column chunk, row phase); a tile row is BLOCK_N*2 contiguous bytes.
template <int BLOCK_N, bool TILE>
DDL_DEVICE void epi_store(uint32_t stg, int etid, const ConvArgs& a, int n0, int m0) {
  constexpr int kPitch = BLOCK_N * 2 + 16;
  constexpr int kVecPerRow = BLOCK_N / 8;
  constexpr int kRowStep = kEpiThreads / kVecPerRow;
  constexpr int kIters = kBlockM / kRowStep;
  const int ch = etid % kVecPerRow;
  const int r0 = etid / kVecPerRow;
  if (n0 + ch * 8 >= a.ldc) return;                       // channel padding of the last N tile (ldc = row width)
  if (a.variant & kDbgNoStore) return;
  uint32_t sp = stg + r0 * kPitch + ch * 16;
  const size_t coff = static_cast<size_t>(n0 + ch * 8);
  if (a.add == nullptr && !(TILE && a.zfill)) {
    // plain stores (every forward launch): nothing but the shared load, the row's address and the store
    if (!TILE) {
      const int rows = a.M - m0;                            // valid rows of this tile (>= kBlockM except in the last one)
      uint4* gp = reinterpret_cast<uint4*>(a.out + static_cast<size_t>(m0 + r0) * a.ldc + coff);
      const size_t gstep = static_cast<size_t>(kRowStep) * a.ldc / 8;      // ldc % 8 == 0 (16-byte rows)
      if (rows >= kBlockM) {
#pragma unroll
        for (int i = 0; i < kIters; ++i) gp[i * gstep] = lds128(sp + i * kRowStep * kPitch);
      } else {
#pragma unroll 1
        for (int r = r0; r < rows; r += kRowStep, sp += kRowStep * kPitch, gp += gstep) *gp = lds128(sp);
      }
    } else {
      __nv_bfloat16* gcol = a.out + coff;
#pragma unroll
      for (int i = 0; i < kIters; ++i) {
        const int m = static_cast<int>(lds32(sp + i * kRowStep * kPitch - ch * 16 + BLOCK_N * 2));
        if (m >= 0) *reinterpret_cast<uint4*>(gcol + static_cast<size_t>(m) * a.ldc) = lds128(sp + i * kRowStep * kPitch);
      }
    }
    return;
  }
#pragma unroll 4
  for (int r = r0; r < kBlockM; r += kRowStep, sp += kRowStep * kPitch) {
    int m;
    if (TILE) m = static_cast<int>(lds32(sp - ch * 16 + BLOCK_N * 2));
    else m = (m0 + r) < a.M ? (m0 + r) : -1;
    if (m < 0) continue;
    uint4 val = lds128(sp);
    const size_t off = static_cast<size_t>(m) * a.ldc + coff;
    if (a.add) {
      uint4 o = *reinterpret_cast<const uint4*>(a.add + off);
      if (a.add_mask) {
        const uint32_t bits = a.add_mask[off >> 3];
        o.x &= ((bits & 1u) ? 0x0000ffffu : 0u) | ((bits & 2u) ? 0xffff0000u : 0u);
        o.y &= ((bits & 4u) ? 0x0000ffffu : 0u) | ((bits & 8u) ? 0xffff0000u : 0u);
        o.z &= ((bits & 16u) ? 0x0000ffffu : 0u) | ((bits & 32u) ? 0xffff0000u : 0u);
        o.w &= ((bits & 64u) ? 0x0000ffffu : 0u) | ((bits & 128u) ? 0xffff0000u : 0u);
      }
      float2 p, q;
      p = unpack_bf16x2(val.x); q = unpack_bf16x2(o.x); val.x = pack_bf16x2(p.x + q.x, p.y + q.y);
      p = unpack_bf16x2(val.y); q = unpack_bf16x2(o.y); val.y = pack_bf16x2(p.x + q.x, p.y + q.y);
      p = unpack_bf16x2(val.z); q = unpack_bf16x2(o.z); val.z = pack_bf16x2(p.x + q.x, p.y + q.y);
      p = unpack_bf16x2(val.w); q = unpack_bf16x2(o.w); val.w = pack_bf16x2(p.x + q.x, p.y + q.y);
    }
    *reinterpret_cast<uint4*>(a.out + off) = val;
    if (TILE && a.zfill) {      // even outH/outW guaranteed by the host: all three siblings exist
      const uint4 z = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(a.out + off + a.ldc) = z;
      *reinterpret_cast<uint4*>(a.out + off + static_cast<size_t>(a.outW) * a.ldc) = z;
      *reinterpret_cast<uint4*>(a.out + off + static_cast<size_t>(a.outW + 1) * a.ldc) = z;
    }
  }
}

// One tile: accumulate, publish, store.
template <int BLOCK_N, bool STATS, bool TILE>
DDL_DEVICE void epi_stats_store(uint32_t stg, uint32_t red, int etid, int ew, const ConvArgs& a, int n0, int m0) {
  if (STATS) {
    StatAcc acc;
    acc.clear();
    epi_stats_accum<BLOCK_N, TILE>(stg, etid, a, n0, m0, acc);
    acc.n0 = n0;
    epi_stats_flush<BLOCK_N>(red, etid, ew, a, acc);
  }
  epi_store<BLOCK_N, TILE>(stg, etid, a, n0, m0);
}

// ---------------------------------------------------------------------------------------------
// fwd / dgrad / plain-GEMM / stem kernel
// ---------------------------------------------------------------------------------------------
// One M x N tile per CTA.  fp8 operands (FP8: e4m3 x e4m3, K-major A and B) use the same 128-byte k-blocks.
template <int N, int FP8, bool BMN>
DDL_DEVICE void mma_kstep(float (&d)[N / 2], uint64_t da, uint64_t db, uint32_t accumulate) {
  if constexpr (FP8 == 2) {
    if constexpr (N == 128) wgmma_e5m2e4m3_n128<0, 0>(d, da, db, accumulate);
    else wgmma_e5m2e4m3_n64<0, 0>(d, da, db, accumulate);
  } else if constexpr (FP8 == 1) {
    if constexpr (N == 128) wgmma_e4m3_n128<0, 0>(d, da, db, accumulate);
    else wgmma_e4m3_n64<0, 0>(d, da, db, accumulate);
  } else {
    if constexpr (N == 128) wgmma_bf16_n128<0, BMN ? 1 : 0>(d, da, db, accumulate);
    else wgmma_bf16_n64<0, BMN ? 1 : 0>(d, da, db, accumulate);
  }
}

template <int BLOCK_N, int MODE, bool STATS, int FP8, bool PERSIST, bool CL>
__global__ void __launch_bounds__(kThreads, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmBh,
                 const __grid_constant__ TmaSet tmAs, ConvArgs a, int n_tiles, int m_tiles) {
  static_assert(!(PERSIST || CL) || mode_a_tma(MODE), "tile loops and CTA pairs need TMA-fed operands");
  const CUtensorMap& tmA = tmAs.m[0];
  using Cfg = FwdCfg<BLOCK_N>;
  constexpr bool kATma = mode_a_tma(MODE);
  constexpr bool kBMn = mode_b_mn(MODE) && FP8 == 0;   // fp8 data gradients read a transposed, K-major weight copy
  constexpr bool kTile = mode_tile(MODE);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nstages = a.stages;
  // [operand ring][epilogue staging tile][barriers (256 B)][statistics scratch]: the staging tile has its own space so
  // that the producers can fill the ring for the next tile while the consumers drain this one
  const uint32_t stg = smem_u32(smem) + nstages * Cfg::kStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + nstages * Cfg::kStageBytes + Cfg::kEpiBytes);
  uint64_t* empty = full + kMaxStages;

  const int warp = threadIdx.x >> 5;
  const int KB = a.KB;
  // work items: (N tile, M tile) — or, for a CTA pair, (N tile, two consecutive M tiles), one per CTA of the pair.
  // A CTA (pair) takes items unit, unit + units, ...; one item per CTA (pair) unless PERSIST.
  const uint32_t rank = CL ? cluster_ctarank() : 0u;
  const int unit = CL ? static_cast<int>(blockIdx.x >> 1) : static_cast<int>(blockIdx.x);
  const int units = CL ? static_cast<int>(gridDim.x >> 1) : static_cast<int>(gridDim.x);
  const int items = n_tiles * (CL ? (m_tiles + 1) / 2 : m_tiles);
  int n0 = 0, m0 = 0, tq0 = 0, tp0 = 0, tn0 = 0;
  auto decode = [&](int item) {
    n0 = (item % n_tiles) * BLOCK_N;
    const int mt = (item / n_tiles) * (CL ? 2 : 1) + static_cast<int>(rank);   // may be m_tiles (odd pair): all rows empty
    m0 = mt * kBlockM;                       // linear modes: rows [m0, m0+128)
    if (kTile) {                             // tile modes: box origin in the output's (w, h, n) space
      int t = mt;
      const int wb = t % a.tiles_w; t /= a.tiles_w;
      const int hb = t % a.tiles_h;
      const int nb = t / a.tiles_h;
      tq0 = wb * a.tw; tp0 = hb * a.th; tn0 = nb * a.tn;
      m0 = 0;
    }
  };

  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&full[s], kATma ? 1u : (kProducerThreads + 1u));
      mbar_init(&empty[s], (kEpiThreads / 32) * (CL ? 2u : 1u));   // one arrival per consumer warp (of both CTAs)
    }
    fence_mbar_init();
  }
  if (warp == kTmaWarp && elect_one()) {
    tma_prefetch_desc(&tmB);
    if (CL) tma_prefetch_desc(&tmBh);
    if (kATma) tma_prefetch_desc(&tmA);
  }
  __syncthreads();
  if (CL) cluster_sync_all();          // the peer's barriers are initialised before anything multicasts into it
  pdl_trigger();      // the next kernel in the stream may start its own preamble
  pdl_wait();         // everything above overlapped the previous kernel's tail; global memory is touched only below

  if (warp >= kProducerWarp0 && warp < kTmaWarp) {
    // =============================== gather producers (one tile) ========================
    decode(unit);
    if (!kATma) {
      const int row = threadIdx.x - kEpiThreads;
      const int m = m0 + row;
      const bool row_ok = m < a.M;
      int img = 0, dh = 0, dw = 0;
      if (row_ok) {
        const int hw = a.dstH * a.dstW;
        img = m / hw;
        const int rem = m - img * hw;
        dh = rem / a.dstW;
        dw = rem - dh * a.dstW;
      }
      int hb, wb;
      if (MODE == kConvDgrad) { hb = dh + a.pad; wb = dw + a.pad_w; }
      else { hb = dh * a.stride - a.pad; wb = dw * a.stride - a.pad_w; }
      const __nv_bfloat16* img_base = a.src + static_cast<size_t>(img) * a.srcH * a.srcW * a.srcC;
      const uint32_t row_off = row * 128u;
      const uint32_t sw = row & 7u;
      int tap_r = 0, tap_s = 0, cc = 0;   // incremental decode of kb -> (r, s, channel chunk)
      int stage = 0;
      uint32_t phase = 0;
      for (int kb = 0; kb < KB; ++kb) {
        mbar_wait(&empty[stage], phase ^ 1u, 17);
        const uint32_t dst = smem_u32(smem + stage * Cfg::kStageBytes) + row_off;
        if (MODE == kConvStem) {
          // k-block = RPK filter rows x SP taps x 4 channels, SP = a.cchunks (padded taps per row)
          const int SP = a.cchunks;
          const int RPK = 16 / SP;           // 64 elements / (SP * 4)
          for (int rr = 0; rr < RPK; ++rr) {
            const int r = kb * RPK + rr;
            const int h = hb + r * a.dil;
            const bool h_ok = row_ok && r < a.R && h >= 0 && h < a.srcH;
            for (int s = 0; s < SP; ++s) {
              const int e = s * RPK + rr;     // 8-byte element index in the 128-byte row: (tap, row-in-block) order
              const int w = wb + s * a.dil;
              const bool ok = h_ok && s < a.S && w >= 0 && w < a.srcW;
              const __nv_bfloat16* src = ok ? img_base + (static_cast<size_t>(h) * a.srcW + w) * 4 : a.src;
              const uint32_t chunk = (e >> 1) ^ sw;
              cp_async_8(dst + (chunk << 4) + ((e & 1) << 3), src, ok);
            }
          }
        } else {
          bool ok;
          int sh, swd;
          if (MODE == kConvDgrad) {
            const int th = hb - tap_r * a.dil, tw = wb - tap_s * a.dil;
            if (a.stride == 1) {
              sh = th; swd = tw;
              ok = row_ok && th >= 0 && th < a.srcH && tw >= 0 && tw < a.srcW;
            } else {
              sh = th / a.stride; swd = tw / a.stride;
              ok = row_ok && th >= 0 && tw >= 0 && (th - sh * a.stride) == 0 && (tw - swd * a.stride) == 0 &&
                   sh < a.srcH && swd < a.srcW;
            }
          } else {
            sh = hb + tap_r * a.dil; swd = wb + tap_s * a.dil;
            ok = row_ok && sh >= 0 && sh < a.srcH && swd >= 0 && swd < a.srcW;
          }
          const __nv_bfloat16* src =
              ok ? img_base + (static_cast<size_t>(sh) * a.srcW + swd) * a.srcC + cc * 64 : a.src;
          const int crem = a.srcC - cc * 64;      // channels left in this tap (last k-block of a tap may be partial)
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const bool okj = ok && j * 8 < crem;
            cp_async_16(dst + ((static_cast<uint32_t>(j) ^ sw) << 4), okj ? src + j * 8 : a.src, okj);
          }
          if (++cc == a.cchunks) { cc = 0; if (++tap_s == a.S) { tap_s = 0; ++tap_r; } }
        }
        cp_async_commit();
        if (kb >= kLag) {
          cp_async_wait<kLag>();
          fence_proxy_async_smem();
          mbar_arrive(&full[(kb - kLag) % nstages]);
        }
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();
      for (int kb = (KB > kLag ? KB - kLag : 0); kb < KB; ++kb) mbar_arrive(&full[kb % nstages]);
    }
  } else if (warp == kTmaWarp) {
    // ================================== TMA producer =====================================
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int item = unit; item < items; item += units) {
        decode(item);
        int tap = 0, cc = 0, tap_r = 0, tap_s = 0;
        const uint32_t a_bytes = kTile ? static_cast<uint32_t>(a.tw * a.th * a.tn) * 128u : kATileBytes;
        for (int kb = 0; kb < KB; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u, 17);
          uint8_t* sA = smem + stage * Cfg::kStageBytes;
          const uint32_t sB = smem_u32(sA + kATileBytes);
          mbar_arrive_expect_tx(&full[stage], Cfg::kBTileBytes + (kATma ? a_bytes : 0u));
          // tap of this k-block: weight tap index + (tile modes) source box offset / source map
          int widx = tap, dh = 0, dw = 0, mapi = 0;
          if (kTile) {
            if (a.ntaps > 0) {
              widx = a.tap_widx[tap]; dh = a.tap_dh[tap]; dw = a.tap_dw[tap]; mapi = a.tap_map[tap];
            } else if (MODE == kConvTileFwd) {
              dh = tap_r * a.dil - a.pad; dw = tap_s * a.dil - a.pad_w;
            } else {
              dh = a.pad - tap_r * a.dil; dw = a.pad_w - tap_s * a.dil;
            }
          }
          const int kcol = FP8 ? 128 : kBlockK;          // elements per 128-byte k-block
          if (CL) {
            // each CTA of the pair loads half of the weight tile and multicasts it into both CTAs
            if (kBMn) {
              tma_load_2d_multicast(sB + rank * 8192u, &tmB, widx * a.ldc + n0 + static_cast<int>(rank) * 64, cc * 64,
                                    &full[stage], 0x3);
            } else {
              tma_load_2d_multicast(sB + rank * (BLOCK_N / 2) * 128u, &tmBh,
                                    mode_stem(MODE) ? kb * kBlockK : widx * a.kstride + cc * kcol,
                                    n0 + static_cast<int>(rank) * (BLOCK_N / 2), &full[stage], 0x3);
            }
          } else if (kBMn) {
            // weights W[co][(r,s,ci)]: K rows = 64 output channels, N = input channels (contiguous)
#pragma unroll
            for (int j = 0; j < BLOCK_N / 64; ++j)
              tma_load_2d(sB + j * 8192, &tmB, widx * a.ldc + n0 + j * 64, cc * 64, &full[stage]);
          } else {
            tma_load_2d(sB, &tmB, mode_stem(MODE) ? kb * kBlockK : widx * a.kstride + cc * kcol, n0, &full[stage]);
          }
          if (MODE == kConvGemm || MODE == kConvGemmDgrad) {
            tma_load_2d(smem_u32(sA), &tmA, kb * kcol, m0, &full[stage]);
          } else if (MODE == kConvStemTma) {
            tma_load_5d(smem_u32(sA), &tmA, 0, kb, tq0, tp0, tn0, &full[stage]);
          } else if (kTile) {
            tma_load_4d(smem_u32(sA), &tmAs.m[mapi], cc * kcol, tq0 + dw, tp0 + dh, tn0, &full[stage]);
          }
          if (++cc == a.cchunks) { cc = 0; ++tap; if (++tap_s == a.S) { tap_s = 0; ++tap_r; } }
          if (++stage == nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
    __syncwarp();
  } else {
    // ============================ consumers: wgmma + epilogue =============================
    // warpgroup g = warps 4g..4g+3 owns accumulator rows [64g, 64g + 64) of the tile
    const int wg = warp >> 2;
    const int lane = threadIdx.x & 31;
    const uint64_t odA0 = smem_desc_sw128(smem_u32(smem) + wg * (kATileBytes / 2), 0, 1024);
    const uint64_t odB0 = kBMn ? smem_desc_sw128(smem_u32(smem) + kATileBytes, 8192, 1024)
                               : smem_desc_sw128(smem_u32(smem) + kATileBytes, 0, 1024);
    const uint32_t oa_lo = static_cast<uint32_t>(odA0), oa_hi = static_cast<uint32_t>(odA0 >> 32);
    const uint32_t ob_lo = static_cast<uint32_t>(odB0), ob_hi = static_cast<uint32_t>(odB0 >> 32);
    // hand a stage back to the producers (of both CTAs of a pair: either may multicast into it next)
    auto release = [&](int s) {
      __syncwarp();
      if (lane == 0) {
        if (CL) {
          const uint32_t local = smem_u32(&empty[s]);
          mbar_arrive_cluster(mapa_shared(local, 0));
          mbar_arrive_cluster(mapa_shared(local, 1));
        } else {
          mbar_arrive(&empty[s]);
        }
      }
    };
    const int etid = threadIdx.x;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    float acc[BLOCK_N / 2];
    int stage = 0;
    uint32_t phase = 0;
    for (int item = unit; item < items; item += units) {
      decode(item);
      int prev = -1;
      for (int kb = 0; kb < KB; ++kb) {
        mbar_wait(&full[stage], phase, 18);
        const uint32_t so = static_cast<uint32_t>(stage) * (Cfg::kStageBytes >> 4);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const uint64_t da = desc_join(oa_lo + so + 2u * k, oa_hi);
          const uint64_t db = desc_join(ob_lo + so + (kBMn ? 128u : 2u) * k, ob_hi);
          mma_kstep<BLOCK_N, FP8, kBMn>(acc, da, db, (kb | k) != 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<1>();               // the previous k-block's MMAs are done: hand its stage back to the producers
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      acc_fence(acc);
      release(prev);
      // every consumer is past the previous tile's stores: the staging tile may be rewritten
      named_bar_sync(1, kEpiThreads);
      auto dest_row = [&](int row) -> int {     // output row of accumulator row `row`, or -1
        if (kTile) {
          const int wl = row % a.tw;
          const int t2 = row / a.tw;
          const int hl = t2 % a.th;
          const int nl = t2 / a.th;
          const bool ok = nl < a.tn && (tn0 + nl) < a.batch && (tp0 + hl) < a.dstH && (tq0 + wl) < a.dstW;
          return ok ? ((tn0 + nl) * a.outH + (tp0 + hl) * a.out_stride + a.out_pa) * a.outW + (tq0 + wl) * a.out_stride +
                          a.out_pb
                    : -1;
        }
        return (m0 + row) < a.M ? (m0 + row) : -1;
      };
      // rows outside the image: exact zeros (keeps the BN sums clean)
      const bool z0 = kTile && dest_row(r0) < 0, z1 = kTile && dest_row(r0 + 8) < 0;
      const float deq = FP8 ? *a.deq_a * *a.deq_b : 1.0f;
      if (!STATS && (a.bias != nullptr || a.relu)) epi_acc_to_stage<BLOCK_N, true>(acc, stg, r0, z0, z1, a, n0, deq);
      else epi_acc_to_stage<BLOCK_N, false>(acc, stg, r0, z0, z1, a, n0, deq);
      // the row's destination index rides in the pad bytes of its staging row (pitch = 2*BLOCK_N + 16)
      if (kTile && etid < kBlockM) sts32(stg + etid * Cfg::kPitch + BLOCK_N * 2, static_cast<uint32_t>(dest_row(etid)));
      named_bar_sync(1, kEpiThreads);
      epi_stats_store<BLOCK_N, STATS, kTile>(stg, smem_u32(full) + 256, etid, warp, a, n0, m0);
    }
  }
  if (CL) cluster_sync_all();          // no CTA leaves while its peer may still multicast into it or arrive on it
}

// ---------------------------------------------------------------------------------------------
// wgrad kernel: dW[co][k] += sum over a pixel range of dY[m][co] * im2col(X)[m][k]
// ---------------------------------------------------------------------------------------------
constexpr int kWgMaxStages = 4;
constexpr int kWgStageBytes = 32768;           // A: 2 x [64 pix][64 co], B: 2 x [64 pix][64 k]
constexpr int kWgPitch = 132;                  // fp32 staging pitch (floats)
constexpr int kWgEpiBytes = kBlockM * kWgPitch * 4;
constexpr int wg_smem_bytes(int stages) {
  return (stages * kWgStageBytes > kWgEpiBytes ? stages * kWgStageBytes : kWgEpiBytes) + 256 + 1024;
}

// SWAP = operand roles exchanged for narrow outputs (Cout tile of 64): the 128-row MMA dimension carries the k
// columns and N = 64 output channels, so no half of the tensor-core tile multiplies zero rows.  The accumulator comes
// out transposed ([k col][co]) and is staged transposed so the global reductions stay row-contiguous.
template <int MODE, bool SWAP>
__global__ void __launch_bounds__(kThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ TmaSet tmXs, WgradArgs a) {
  const CUtensorMap& tmX = tmXs.m[0];
  constexpr bool kXTma = (MODE == kConvGemm || MODE == kConvTileFwd || MODE == kConvStemTma);
  constexpr bool kTile = (MODE == kConvTileFwd || MODE == kConvStemTma);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int nstages = a.stages;
  const int pipe_bytes = nstages * kWgStageBytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + (pipe_bytes > kWgEpiBytes ? pipe_bytes : kWgEpiBytes));
  uint64_t* empty = full + kWgMaxStages;

  const int warp = threadIdx.x >> 5;
  const int col0 = blockIdx.x * 128;          // first k column of this tile
  constexpr int kCoTile = SWAP ? 64 : 128;
  const int co0 = blockIdx.y * kCoTile;       // first output channel of this tile
  const int kb_begin = blockIdx.z * a.kb_per_split;
  const int kb_end = min(kb_begin + a.kb_per_split, a.total_kb);
  const int KB = kb_end - kb_begin;
  if (KB <= 0) return;                         // uniform per CTA

  if (threadIdx.x == 0) {
    for (int s = 0; s < nstages; ++s) {
      mbar_init(&full[s], kXTma ? 1u : (kProducerThreads + 1u));
      mbar_init(&empty[s], kEpiThreads / 32);
    }
    fence_mbar_init();
  }
  if (warp == kTmaWarp && elect_one()) {
    tma_prefetch_desc(&tmDy);
    if (kXTma) tma_prefetch_desc(&tmX);
  }
  if (kTile) {
    // pixel boxes may hold fewer than 64 rows: the unused K rows of EVERY operand chunk must read as zero
    const int rows = a.tw * a.th * a.tn;
    const int tail16 = (64 - rows) * 8;        // 16-byte units per 8 KB chunk
    for (int st = 0; st < nstages; ++st)
      for (int chunk = 0; chunk < 4; ++chunk) {
        uint4* base = reinterpret_cast<uint4*>(smem + st * kWgStageBytes + chunk * 8192 + rows * 128);
        for (int i = threadIdx.x; i < tail16; i += kThreads) base[i] = make_uint4(0, 0, 0, 0);
      }
    fence_proxy_async_smem();
  }
  __syncthreads();

  if (warp >= kProducerWarp0 && warp < kTmaWarp) {
    if (!kXTma) {
      const int t = threadIdx.x - kEpiThreads;
      const int chunk = t >> 6;                // which 64-column half of the B tile
      const int row = t & 63;                  // pixel row inside the k-block
      const int colc = col0 + chunk * 64;      // first k column of my chunk
      const bool col_ok = colc < a.ncols;
      int tap_r = 0, tap_s = 0, c_off = 0;
      if (!mode_stem(MODE)) {
        const int tap = colc / a.Cpad;          // columns live in the padded (tap, Cpad) space
        c_off = colc - tap * a.Cpad;
        tap_r = tap / a.S;
        tap_s = tap - tap_r * a.S;
      }
      const int crem = a.C - c_off;             // real channels left in this tap
      const uint32_t row_off = 16384u + chunk * 8192u + row * 128u;
      const uint32_t sw = row & 7u;
      const int pq = a.P * a.Q;
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < KB; ++i) {
        mbar_wait(&empty[stage], phase ^ 1u, 65);
        const uint32_t dst = smem_u32(smem + stage * kWgStageBytes) + row_off;
        const int m = (kb_begin + i) * 64 + row;
        const bool m_ok = col_ok && m < a.M;
        int img = 0, p = 0, q = 0;
        if (m_ok) {
          img = m / pq;
          const int rem = m - img * pq;
          p = rem / a.Q;
          q = rem - p * a.Q;
        }
        const int hb = p * a.stride - a.pad, wb = q * a.stride - a.pad_w;
        const __nv_bfloat16* img_base = a.x + static_cast<size_t>(img) * a.H * a.W * a.C;
        if (MODE == kConvStem) {
          const int SP = a.cchunks, RPK = 16 / SP;
          const int kbk = colc / 64;            // which k-block of the stem's packed K
          for (int rr = 0; rr < RPK; ++rr) {
            const int r = kbk * RPK + rr;
            const int h = hb + r * a.dil;
            const bool h_ok = m_ok && r < a.R && h >= 0 && h < a.H;
            for (int s = 0; s < SP; ++s) {
              const int e = s * RPK + rr;
              const int w = wb + s * a.dil;
              const bool ok = h_ok && s < a.S && w >= 0 && w < a.W;
              const __nv_bfloat16* src = ok ? img_base + (static_cast<size_t>(h) * a.W + w) * 4 : a.x;
              cp_async_8(dst + (((e >> 1) ^ sw) << 4) + ((e & 1) << 3), src, ok);
            }
          }
        } else {
          const int h = hb + tap_r * a.dil, w = wb + tap_s * a.dil;
          const bool ok = m_ok && h >= 0 && h < a.H && w >= 0 && w < a.W;
          const __nv_bfloat16* src = ok ? img_base + (static_cast<size_t>(h) * a.W + w) * a.C + c_off : a.x;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const bool okj = ok && j * 8 < crem;
            cp_async_16(dst + ((static_cast<uint32_t>(j) ^ sw) << 4), okj ? src + j * 8 : a.x, okj);
          }
        }
        cp_async_commit();
        if (i >= kLag) {
          cp_async_wait<kLag>();
          fence_proxy_async_smem();
          mbar_arrive(&full[(i - kLag) % nstages]);
        }
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
      cp_async_wait<0>();
      fence_proxy_async_smem();
      for (int i = (KB > kLag ? KB - kLag : 0); i < KB; ++i) mbar_arrive(&full[i % nstages]);
    }
  } else if (warp == kTmaWarp) {
    if (elect_one()) {
      // taps / channel offsets of the two 64-column chunks of the B tile (tile mode)
      int tdh[2] = {0, 0}, tdw[2] = {0, 0}, tmap[2] = {0, 0}, tc0[2] = {0, 0};
      if (kTile && MODE != kConvStemTma) {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int colc = col0 + j * 64;
          const int tap = colc / a.Cpad;
          tc0[j] = colc - tap * a.Cpad;
          const int r = tap / a.S, sx = tap - r * a.S;
          const int oh = r * a.dil - a.pad, ow = sx * a.dil - a.pad_w;
          if (a.stride == 1) {
            tdh[j] = oh; tdw[j] = ow;
          } else {               // stride-2 source: box comes from the (pa, pb) phase sub-image
            const int st = a.stride;
            const int pa = ((oh % st) + st) % st, pb = ((ow % st) + st) % st;
            tdh[j] = (oh - pa) / st; tdw[j] = (ow - pb) / st;
            tmap[j] = pa * st + pb;
          }
        }
      }
      const uint32_t box_bytes = kTile ? static_cast<uint32_t>(a.tw * a.th * a.tn) * 128u : 8192u;
      int stage = 0;
      uint32_t phase = 0;
      for (int i = 0; i < KB; ++i) {
        mbar_wait(&empty[stage], phase ^ 1u, 65);
        const uint32_t sA = smem_u32(smem + stage * kWgStageBytes);
        if (kTile) {
          int t = kb_begin + i;
          const int wb = t % a.tiles_w; t /= a.tiles_w;
          const int hb = t % a.tiles_h;
          const int nb = t / a.tiles_h;
          const int q0 = wb * a.tw, p0 = hb * a.th, n0 = nb * a.tn;
          const bool second = (col0 + 64) < a.ncols;
          mbar_arrive_expect_tx(&full[stage], box_bytes * ((second ? 4u : 3u) - (SWAP ? 1u : 0u)));
          tma_load_4d(sA, &tmDy, co0, q0, p0, n0, &full[stage]);
          if (!SWAP) tma_load_4d(sA + 8192, &tmDy, co0 + 64, q0, p0, n0, &full[stage]);
          if (MODE == kConvStemTma) {
            // k-block (col0 / 64 + j) of the packed stem K = one box of the row-interleaved image
            tma_load_5d(sA + 16384, &tmXs.m[0], 0, col0 / 64, q0, p0, n0, &full[stage]);
            if (second) tma_load_5d(sA + 24576, &tmXs.m[0], 0, col0 / 64 + 1, q0, p0, n0, &full[stage]);
          } else {
            tma_load_4d(sA + 16384, &tmXs.m[tmap[0]], tc0[0], q0 + tdw[0], p0 + tdh[0], n0, &full[stage]);
            if (second) tma_load_4d(sA + 24576, &tmXs.m[tmap[1]], tc0[1], q0 + tdw[1], p0 + tdh[1], n0, &full[stage]);
          }
        } else {
          const int m = (kb_begin + i) * 64;
          mbar_arrive_expect_tx(&full[stage], (SWAP ? 8192u : 16384u) + (kXTma ? 16384u : 0u));
          tma_load_2d(sA, &tmDy, co0, m, &full[stage]);
          if (!SWAP) tma_load_2d(sA + 8192, &tmDy, co0 + 64, m, &full[stage]);
          if (kXTma) {
            tma_load_2d(sA + 16384, &tmX, col0, m, &full[stage]);
            tma_load_2d(sA + 24576, &tmX, col0 + 64, m, &full[stage]);
          }
        }
        if (++stage == nstages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // consumers: warpgroup g multiplies the g-th 64-wide chunk of the M operand (both operands MN-major)
    constexpr int kN = SWAP ? 64 : 128;
    const int wg = warp >> 2;
    const int lane = threadIdx.x & 31;
    float acc[kN / 2];
#pragma unroll
    for (int i = 0; i < kN / 2; ++i) acc[i] = 0.f;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int i = 0; i < KB; ++i) {
      mbar_wait(&full[stage], phase, 66);
      const uint32_t sDy = smem_u32(smem + stage * kWgStageBytes);
      const uint32_t sX = sDy + 16384;
      const uint32_t sA = (SWAP ? sX : sDy) + wg * 8192;   // M operand: 128 rows = two 64-wide MN-major chunks 8 KB apart
      const uint32_t sB = SWAP ? sDy : sX;                 // N operand (SWAP: one 64-channel chunk of dY)
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const uint64_t da = smem_desc_sw128(sA + k * 2048, 8192, 1024);
        const uint64_t db = smem_desc_sw128(sB + k * 2048, 8192, 1024);
        if constexpr (SWAP) wgmma_bf16_n64<1, 1>(acc, da, db, (i | k) != 0 ? 1u : 0u);
        else wgmma_bf16_n128<1, 1>(acc, da, db, (i | k) != 0 ? 1u : 0u);
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty[prev]);
      }
      prev = stage;
      if (++stage == nstages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
    acc_fence(acc);
    named_bar_sync(1, kEpiThreads);
    // epilogue: registers -> fp32 staging -> coalesced vector reductions into the gradient arena
    float* stg = reinterpret_cast<float*>(smem);
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      if (SWAP) {
        // accumulator row = k column, accumulator column = output channel: stage as [co][k col]
        stg[c * kWgPitch + r0] = acc[4 * j];
        stg[(c + 1) * kWgPitch + r0] = acc[4 * j + 1];
        stg[c * kWgPitch + r0 + 8] = acc[4 * j + 2];
        stg[(c + 1) * kWgPitch + r0 + 8] = acc[4 * j + 3];
      } else {
        *reinterpret_cast<float2*>(stg + r0 * kWgPitch + c) = make_float2(acc[4 * j], acc[4 * j + 1]);
        *reinterpret_cast<float2*>(stg + (r0 + 8) * kWgPitch + c) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
      }
    }
    named_bar_sync(1, kEpiThreads);
    const int vc = col0 + lane * 4;                    // column in the padded (tap, Cpad) space
    const int vtap = vc / a.Cpad;
    const int vch = vc - vtap * a.Cpad;
    if (vc < a.ncols && vch < a.Cw) {                  // channel padding of a tap has no dw column
      const int c = vtap * a.Cw + vch;
      for (int r = warp; r < kCoTile; r += kEpiThreads / 32) {
        const int co = co0 + r;
        if (co < a.Cout) {
          const float4 val = *reinterpret_cast<const float4*>(stg + r * kWgPitch + lane * 4);
          red_add_f32x4(a.dw + static_cast<size_t>(co) * a.ldw + c, val.x, val.y, val.z, val.w);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// host side: tensor maps + launchers
// ---------------------------------------------------------------------------------------------
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                   CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = []() -> EncodeTiledFn {
    void* lib = dlopen("libcuda.so.1", RTLD_NOW | RTLD_GLOBAL);
    if (!lib) return nullptr;
    return reinterpret_cast<EncodeTiledFn>(dlsym(lib, "cuTensorMapEncodeTiled"));
  }();
  return fn;
}

// 2-D bf16 row-major matrix [rows][cols] (cols contiguous), box = {box_cols, box_rows}, 128B swizzle.
// `esize` = element size in bytes: 2 = bf16, 1 = fp8 (maps over bytes; a 128-byte swizzle row is 128 elements then).
bool make_map_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint64_t row_stride_elems,
                 uint32_t box_cols, uint32_t box_rows, int esize = 2) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {row_stride_elems * static_cast<uint64_t>(esize)};
  cuuint32_t box[2] = {box_cols, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = fn(map, esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// 4-D NHWC bf16 activation [N][H][W][C]; box = {64 channels, tw, th, tn}; out-of-bounds -> zeros.
bool make_map_nhwc(CUtensorMap* map, const void* base, int N, int H, int W, int C, int tw, int th, int tn,
                   int esize = 2) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t es = static_cast<cuuint64_t>(esize);
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(W), static_cast<cuuint64_t>(H),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(C) * es, static_cast<cuuint64_t>(W) * C * es,
                           static_cast<cuuint64_t>(H) * W * C * es};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(128 / esize), static_cast<cuuint32_t>(tw), static_cast<cuuint32_t>(th),
                       static_cast<cuuint32_t>(tn)};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// Phase (pa, pb) sub-image of a stride-`st` NHWC source: X[n][st*i + pa][st*j + pb][c] as a dense 4-D map.
bool make_map_nhwc_phase(CUtensorMap* map, const void* base, int N, int H, int W, int C, int st, int pa, int pb,
                         int tw, int th, int tn, int esize = 2) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const int Hp = (H - pa + st - 1) / st, Wp = (W - pb + st - 1) / st;
  if (Hp <= 0 || Wp <= 0) return make_map_nhwc(map, base, N, H, W, C, tw, th, tn, esize);   // never referenced
  const cuuint64_t es = static_cast<cuuint64_t>(esize);
  const char* b = static_cast<const char*>(base) + (static_cast<size_t>(pa) * W + pb) * C * es;
  cuuint64_t dims[4] = {static_cast<cuuint64_t>(C), static_cast<cuuint64_t>(Wp), static_cast<cuuint64_t>(Hp),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t strides[3] = {static_cast<cuuint64_t>(st) * C * es, static_cast<cuuint64_t>(st) * W * C * es,
                           static_cast<cuuint64_t>(H) * W * C * es};
  cuuint32_t box[4] = {static_cast<cuuint32_t>(128 / esize), static_cast<cuuint32_t>(tw), static_cast<cuuint32_t>(th),
                       static_cast<cuuint32_t>(tn)};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUresult r = fn(map, esize == 1 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<char*>(b), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

// Stem operand map over the zero-padded, G-row-interleaved image [N][Hp][Wp][G][4] written by pad_nhwc4
// (G = RPK filter rows per k-block): the k-block j of output pixel (n, p, q) is the 128 contiguous bytes at
// (row stride*p + G*j, col stride*q).  5-D map (64 elements | k-block | out col | out row | image) whose dimensions
// overlap in memory; box = {64, 1, tw, th, tn}.
bool make_map_stem5d(CUtensorMap* map, const void* base, int N, int Hp, int Wp, int P, int Q, int stride, int G, int KB,
                     int tw, int th, int tn) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t pitch = static_cast<cuuint64_t>(Wp) * G * 8;          // bytes per buffer row
  cuuint64_t dims[5] = {64, static_cast<cuuint64_t>(KB), static_cast<cuuint64_t>(Q), static_cast<cuuint64_t>(P),
                        static_cast<cuuint64_t>(N)};
  cuuint64_t strides[4] = {pitch * G, static_cast<cuuint64_t>(stride) * G * 8, pitch * stride, pitch * Hp};
  cuuint32_t box[5] = {64, 1, static_cast<cuuint32_t>(tw), static_cast<cuuint32_t>(th), static_cast<cuuint32_t>(tn)};
  cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  for (int i = 0; i < 4; ++i)
    if (strides[i] % 16 != 0) return false;
  CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS;
}

inline int stem_sp(int S) { return S <= 4 ? 4 : (S <= 8 ? 8 : 16); }

inline int floor_div(int a, int b) { return (a >= 0) ? a / b : -((-a + b - 1) / b); }

int g_num_sms = 0;

int num_sms() {
  if (g_num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&g_num_sms, cudaDevAttrMultiProcessorCount, dev);
    if (g_num_sms <= 0) g_num_sms = 132;
  }
  return g_num_sms;
}

template <int BLOCK_N, int MODE, bool STATS, int FP8, bool PERSIST, bool CL>
cudaError_t launch_fwd_t(const CUtensorMap& tmB, const CUtensorMap& tmBh, const TmaSet& tmA, const ConvArgs& a,
                         int n_total, int m_tiles, cudaStream_t stream) {
  using Cfg = FwdCfg<BLOCK_N>;
  auto kern = conv_gemm_kernel<BLOCK_N, MODE, STATS, FP8, PERSIST, CL>;
  static bool configured = false;
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                         Cfg::smem_bytes(Cfg::kMaxStagesN));
    if (e != cudaSuccess) return e;
    if (CL) {
      e = cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 0);
      if (e != cudaSuccess) return e;
    }
    configured = true;
  }
  const int n_tiles = n_total / BLOCK_N;
  const long long items = static_cast<long long>(n_tiles) * (CL ? (m_tiles + 1) / 2 : m_tiles);
  long long units = items;
  if (PERSIST) {                                   // one CTA (pair) per SM (pair), each walking several tiles
    const long long slots = CL ? num_sms() / 2 : num_sms();
    if (units > slots) units = slots;
  }
  const long long grid = units * (CL ? 2 : 1);
  if (grid > 0x7fffffffLL) return cudaErrorInvalidValue;
  return launch_pdl(kern, dim3(static_cast<unsigned>(grid)), dim3(kThreads), Cfg::smem_bytes(a.stages), stream,
                    CL ? 2 : 1, tmB, tmBh, tmA, a, n_tiles, m_tiles);
}

// Variant word (ConvArgs::variant; 0 = built-in policy).  The Python layer autotunes it per layer shape on first use
// (ops/native.py: the analogue of the reference's `cudnn.benchmark = True`, pytorch_synthetic_benchmark.py:57).
//   bits 0-3  kernel: 1 = one tile per CTA, 2 = persistent (one CTA per SM walking tiles)
//   bit  8    CTA pairs (clusters of two along M) that share the weight tile by TMA multicast
// (3 = the deep-ring kernel of tensor-memory GPUs has no sm_90 form and is rejected)
constexpr int kVarOneTile = 1, kVarPersistent = 2;

// Pipeline-depth policy: one CTA per SM, so the ring is as deep as the shared memory allows (TMA round trips stay
// covered on long-K layers).  g_force_stages (tuning hook) overrides.
int g_force_stages = 0;
int g_wgrad_swap = 1;       // tuning hook: 0 disables the operand-role swap of narrow-output wgrad tiles
int g_persistent = 1;       // tuning hook: 0 = never the persistent kernel, 1 = policy (variant word), 2 = always
int g_cluster = 0;          // tuning hook: != 0 = the persistent kernel runs as CTA pairs wherever they apply
int g_deep = 1;             // tuning hook: 0 = never, 1 = policy, 2 = persistent CTA pairs wherever they apply,
                            //   3 / 4 = persistent single CTAs (one CTA per SM with the deepest ring, as the deep-ring
                            //   kernel of tensor-memory GPUs; tiles are at most 128 wide on sm_90)

template <int BLOCK_N, int MODE>
int pick_stages(int KB) {
  const int max_s = FwdCfg<BLOCK_N>::kMaxStagesN;
  int s = g_force_stages > 0 ? g_force_stages : max_s;
  if (s > max_s) s = max_s;
  if (s > KB) s = KB;
  // a consumer releases a stage only after issuing the next k-block's MMAs, and a gather producer completes a stage
  // only kLag k-blocks after filling it: a ring that wraps needs 2 (TMA) / kLag + 2 (gather) stages not to dead-lock
  const int min_s = mode_a_tma(MODE) ? 2 : kLag + 2;
  if (KB > s && s < min_s) s = min_s;
  return s < 1 ? 1 : s;
}

template <int MODE>
constexpr bool mode_persist() {
  return MODE == kConvGemm || MODE == kConvTileFwd || MODE == kConvTileDgrad || MODE == kConvGemmDgrad;
}

template <int BLOCK_N, int MODE>
cudaError_t launch_bn(const CUtensorMap& tmB, const CUtensorMap& tmBh, const TmaSet& tmA, ConvArgs a, int n_total,
                      int m_tiles, bool stats, bool persistent, bool pair, cudaStream_t stream) {
  a.stages = pick_stages<BLOCK_N, MODE>(a.KB);
#define DDL_FWD(FP8, PER, CLU)                                                                                    \
  return stats ? launch_fwd_t<BLOCK_N, MODE, true, FP8, PER, CLU>(tmB, tmBh, tmA, a, n_total, m_tiles, stream)   \
               : launch_fwd_t<BLOCK_N, MODE, false, FP8, PER, CLU>(tmB, tmBh, tmA, a, n_total, m_tiles, stream)
  if (a.fp8) {
    // fp8 wgmma reads K-major operands only: e4m3 x e4m3 forward GEMM / tile modes, e5m2 x e4m3 data gradients on the
    // transposed weight copy; one tile per CTA
    if constexpr (MODE == kConvGemm || MODE == kConvTileFwd) {
      if (a.fp8 == 1) { DDL_FWD(1, false, false); }
    } else if constexpr (MODE == kConvGemmDgrad || MODE == kConvTileDgrad) {
      if (a.fp8 == 2) { DDL_FWD(2, false, false); }
    }
    return cudaErrorInvalidValue;
  }
  if constexpr (mode_persist<MODE>()) {
    if (persistent && pair) { DDL_FWD(0, true, true); }
    if (persistent) { DDL_FWD(0, true, false); }
  }
  DDL_FWD(0, false, false);
#undef DDL_FWD
}

template <int MODE>
cudaError_t launch_fwd_mode(const CUtensorMap& tmB, const CUtensorMap& tmBh, const TmaSet& tmA, const ConvArgs& a,
                            int n_total, int m_tiles, bool stats, cudaStream_t stream) {
  const int var_kind = a.variant & 0xf;
  const bool var_pair = ((a.variant >> 8) & 1) != 0;
  if (var_kind != 0 && var_kind != kVarOneTile && var_kind != kVarPersistent) return cudaErrorInvalidValue;
  const int bn = (n_total % 128 == 0) ? 128 : 64;
  if (n_total % 64 != 0) return cudaErrorInvalidValue;
  // pairs need two M tiles and a weight tile that splits into two loadable halves (MN-major: two 64-column boxes)
  const bool pair_ok = m_tiles >= 2 && (!mode_b_mn(MODE) || bn == 128);
  bool persistent = false, pair = false;
  if (var_kind == kVarPersistent) {
    if (!mode_persist<MODE>() || a.fp8 || (var_pair && !pair_ok)) return cudaErrorInvalidValue;
    persistent = true;
    pair = var_pair;
  } else if (var_kind == 0 && mode_persist<MODE>() && !a.fp8) {
    if (g_deep >= 2) {
      persistent = true;
      pair = g_deep == 2 && pair_ok;
    } else if (g_persistent == 2) {
      persistent = true;
      pair = g_cluster != 0 && pair_ok;
    }
  } else if (var_pair) {
    return cudaErrorInvalidValue;
  }
  if (bn == 128) return launch_bn<128, MODE>(tmB, tmBh, tmA, a, n_total, m_tiles, stats, persistent, pair, stream);
  return launch_bn<64, MODE>(tmB, tmBh, tmA, a, n_total, m_tiles, stats, persistent, pair, stream);
}

}  // namespace

// {abort flag, site, block, thread, parity} of the first mbarrier wait that timed out since the last call; clears it.
cudaError_t conv_timeout_info(unsigned int out[8]) {
  cudaError_t e = cudaMemcpyFromSymbol(out, tc::g_mbar_diag, sizeof(unsigned int) * 8);
  if (e != cudaSuccess) return e;
  if (out[0] != 0u) {
    unsigned int zero[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    e = cudaMemcpyToSymbol(tc::g_mbar_diag, zero, sizeof(zero));
  }
  return e;
}

void set_conv_force_stages(int s) { g_force_stages = s; }
void set_wgrad_swap(int on) { g_wgrad_swap = on; }
void set_conv_persistent(int on) { g_persistent = on; }
void set_conv_cluster(int on) { g_cluster = on; }
void set_conv_deep(int on) { g_deep = on; }
void set_conv_wait_hint(int ns) {
  const unsigned int v = ns > 0 ? static_cast<unsigned int>(ns) : 0u;
  cudaMemcpyToSymbol(tc::c_wait_hint_ns, &v, sizeof(v));
}
void pdl_early_bn(int early);       // bn_act.cu's copy of c_pdl_early
void set_pdl(int on) {
  g_pdl = on;
  const int trig = on == 2 ? 1 : (on >= 3 ? 2 : 0);
  cudaMemcpyToSymbol(c_pdl_trigger, &trig, sizeof(int));
  pdl_early_bn(trig);
}

// `w` is the bf16 weight matrix [n_total][KB*64] (fwd / gemm / stem) or [Cout][R*S*Cin] (dgrad modes).
// `a_matrix`: the A operand for the TMA-A modes (2-D matrix [M][a_cols], or the NHWC tensor in tile modes).
cudaError_t launch_conv_gemm(int mode, const ConvArgs& a_in, const void* w, int w_rows, int w_cols, int n_total,
                             const void* a_matrix, int a_cols, cudaStream_t stream) {
  ConvArgs a = a_in;
  CUtensorMap tmB;
  TmaSet tmA;
  const int bn = (n_total % 128 == 0) ? 128 : 64;
  if (n_total % 64 != 0) return cudaErrorInvalidValue;
  const int es = a.fp8 ? 1 : 2;                   // operand element size (bytes)
  const uint32_t kcols = 128u / es;               // elements in a 128-byte swizzle row
  if (a.fp8) {
    // fp8 operands, K-major, 128-element k-blocks: e4m3 x e4m3 forward (GEMM / tile modes) or e5m2 x e4m3 data
    // gradient (GEMM / tile modes; `w` is then the transposed weight copy [Cin][R*S*Cout], a.kstride = Cout)
    const bool fwd = a.fp8 == 1 && (mode == kConvGemm || mode == kConvTileFwd);
    const bool dgrad = a.fp8 == 2 && (mode == kConvGemmDgrad || mode == kConvTileDgrad);
    if (!(fwd || dgrad) || a.deq_a == nullptr || a.deq_b == nullptr || (dgrad && n_total % 128 != 0))
      return cudaErrorInvalidValue;
  }
  CUtensorMap tmBh;                 // K-major weights: half-height box (one CTA's share of a CTA-pair tile)
  if (mode_b_mn(mode) && !a.fp8) {
    if (!make_map_2d(&tmB, w, w_rows, w_cols, w_cols, kcols, kcols, es)) return cudaErrorUnknown;
    tmBh = tmB;
  } else {
    if (!make_map_2d(&tmB, w, w_rows, w_cols, w_cols, kcols, bn, es)) return cudaErrorUnknown;
    if (!make_map_2d(&tmBh, w, w_rows, w_cols, w_cols, kcols, bn / 2, es)) return cudaErrorUnknown;
  }
  a.ntaps = 0;
  a.outH = a.dstH; a.outW = a.dstW; a.out_stride = 1; a.out_pa = 0; a.out_pb = 0;
  const int want_zfill = a.zfill;
  a.zfill = 0;
  int m_tiles = (a.M + kBlockM - 1) / kBlockM;
  const bool stats = a.sum != nullptr;
  auto dispatch = [&](const ConvArgs& args, int tiles) -> cudaError_t {
    switch (mode) {
      case kConvFwd: return launch_fwd_mode<kConvFwd>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvDgrad: return launch_fwd_mode<kConvDgrad>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvGemm: return launch_fwd_mode<kConvGemm>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvStem: return launch_fwd_mode<kConvStem>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvTileFwd: return launch_fwd_mode<kConvTileFwd>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvTileDgrad: return launch_fwd_mode<kConvTileDgrad>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvGemmDgrad: return launch_fwd_mode<kConvGemmDgrad>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      case kConvStemTma: return launch_fwd_mode<kConvStemTma>(tmB, tmBh, tmA, args, n_total, tiles, stats, stream);
      default: return cudaErrorInvalidValue;
    }
  };
  if (mode == kConvGemm || mode == kConvGemmDgrad) {
    if (!make_map_2d(&tmA.m[0], a_matrix, a.M, a_cols, a_cols, kcols, 128, es)) return cudaErrorUnknown;
    for (int i = 1; i < 4; ++i) tmA.m[i] = tmA.m[0];
    return dispatch(a, m_tiles);
  }
  if (!mode_tile(mode)) {
    for (int i = 0; i < 4; ++i) tmA.m[i] = tmB;
    return dispatch(a, m_tiles);
  }
  // ---------------- tile modes ----------------
  if (a.tw * a.th * a.tn > 128 || a.tw < 1 || a.th < 1 || a.tn < 1) return cudaErrorInvalidValue;
  const int st = a.stride;
  auto set_tiles = [&](ConvArgs& x) {
    x.tiles_w = (x.dstW + x.tw - 1) / x.tw;
    x.tiles_h = (x.dstH + x.th - 1) / x.th;
    return x.tiles_w * x.tiles_h * ((x.batch + x.tn - 1) / x.tn);
  };
  if (mode == kConvStemTma) {
    // a.srcH x a.srcW is the PADDED image; the k-block geometry follows from the filter width (see stem_geometry)
    if (a.S > 16) return cudaErrorInvalidValue;
    const int SP = stem_sp(a.S), RPK = 16 / SP;
    if (!make_map_stem5d(&tmA.m[0], a_matrix, a.batch, a.srcH, a.srcW, a.dstH, a.dstW, st, RPK, a.KB, a.tw, a.th, a.tn))
      return cudaErrorInvalidValue;
    for (int i = 1; i < 4; ++i) tmA.m[i] = tmA.m[0];
    a.cchunks = RPK;
    return dispatch(a, set_tiles(a));
  }
  if (st == 1) {
    if (!make_map_nhwc(&tmA.m[0], a_matrix, a.batch, a.srcH, a.srcW, a.srcC, a.tw, a.th, a.tn, es)) return cudaErrorUnknown;
    for (int i = 1; i < 4; ++i) tmA.m[i] = tmA.m[0];
    return dispatch(a, set_tiles(a));
  }
  if (st != 2 || a.R * a.S > 16) return cudaErrorInvalidValue;
  if (mode == kConvTileFwd) {
    // stride-2 forward: every filter tap reads a dense box of one of the four 2x2 phase sub-images of x
    for (int pa = 0; pa < 2; ++pa)
      for (int pb = 0; pb < 2; ++pb)
        if (!make_map_nhwc_phase(&tmA.m[pa * 2 + pb], a_matrix, a.batch, a.srcH, a.srcW, a.srcC, 2, pa, pb, a.tw, a.th,
                                 a.tn, es))
          return cudaErrorUnknown;
    a.ntaps = a.R * a.S;
    for (int r = 0; r < a.R; ++r)
      for (int sx = 0; sx < a.S; ++sx) {
        const int t = r * a.S + sx;
        const int oh = r * a.dil - a.pad, ow = sx * a.dil - a.pad_w;
        const int pa = ((oh % 2) + 2) % 2, pb = ((ow % 2) + 2) % 2;
        a.tap_dh[t] = static_cast<signed char>(floor_div(oh, 2));
        a.tap_dw[t] = static_cast<signed char>(floor_div(ow, 2));
        a.tap_map[t] = static_cast<signed char>(pa * 2 + pb);
        a.tap_widx[t] = static_cast<signed char>(t);
      }
    return dispatch(a, set_tiles(a));
  }
  // stride-2 data gradient: four stride-1 problems, one per output phase (pa, pb) of dx; each is a conv of dy
  // with the subset of taps of matching parity, scattered to dx[2i+pa][2j+pb].  Phases with no tap stay as the
  // caller initialised them (the Python wrapper zero-fills dx when such phases exist).
  if (!make_map_nhwc(&tmA.m[0], a_matrix, a.batch, a.srcH, a.srcW, a.srcC, a.tw, a.th, a.tn, es)) return cudaErrorUnknown;
  for (int i = 1; i < 4; ++i) tmA.m[i] = tmA.m[0];
  const int fullH = a.dstH, fullW = a.dstW;
  for (int pa = 0; pa < 2; ++pa)
    for (int pb = 0; pb < 2; ++pb) {
      ConvArgs p = a;
      p.dstH = (fullH - pa + 1) / 2;
      p.dstW = (fullW - pb + 1) / 2;
      if (p.dstH <= 0 || p.dstW <= 0) continue;
      p.outH = fullH; p.outW = fullW; p.out_stride = 2; p.out_pa = pa; p.out_pb = pb;
      int nt = 0;
      for (int r = 0; r < a.R; ++r) {
        const int th_ = pa + a.pad - r * a.dil;
        if (((th_ % 2) + 2) % 2 != 0) continue;
        for (int sx = 0; sx < a.S; ++sx) {
          const int tw_ = pb + a.pad_w - sx * a.dil;
          if (((tw_ % 2) + 2) % 2 != 0) continue;
          p.tap_dh[nt] = static_cast<signed char>(floor_div(th_, 2));
          p.tap_dw[nt] = static_cast<signed char>(floor_div(tw_, 2));
          p.tap_map[nt] = 0;
          p.tap_widx[nt] = static_cast<signed char>(r * a.S + sx);
          ++nt;
        }
      }
      if (nt == 0) continue;
      p.zfill = (want_zfill && pa == 0 && pb == 0 && fullH % 2 == 0 && fullW % 2 == 0) ? 1 : 0;
      p.ntaps = nt;
      p.KB = nt * a.cchunks;
      cudaError_t e = dispatch(p, set_tiles(p));
      if (e != cudaSuccess) return e;
    }
  return cudaSuccess;
}

cudaError_t launch_conv_wgrad(const WgradArgs& a_in, const void* dy, const void* x_matrix, int splits,
                              cudaStream_t stream) {
  WgradArgs a = a_in;
  CUtensorMap tmDy;
  TmaSet tmX;
  if (a.mode == kConvTileFwd || a.mode == kConvStemTma) {
    if (a.tw * a.th * a.tn > 64 || a.tw < 1 || a.th < 1 || a.tn < 1) return cudaErrorInvalidValue;
    if (!make_map_nhwc(&tmDy, dy, a.batch, a.P, a.Q, a.dy_ld, a.tw, a.th, a.tn)) return cudaErrorUnknown;
    if (a.mode == kConvStemTma) {
      // a.H x a.W is the PADDED image, a.cchunks = SP, a.ncols = KB * 64
      if (a.cchunks < 4) return cudaErrorInvalidValue;
      const int RPK = 16 / a.cchunks;
      if (!make_map_stem5d(&tmX.m[0], x_matrix, a.batch, a.H, a.W, a.P, a.Q, a.stride, RPK, a.ncols / 64, a.tw, a.th,
                           a.tn))
        return cudaErrorInvalidValue;
      for (int i = 1; i < 4; ++i) tmX.m[i] = tmX.m[0];
    } else if (a.stride == 1) {
      if (!make_map_nhwc(&tmX.m[0], x_matrix, a.batch, a.H, a.W, a.C, a.tw, a.th, a.tn)) return cudaErrorUnknown;
      for (int i = 1; i < 4; ++i) tmX.m[i] = tmX.m[0];
    } else if (a.stride == 2) {
      for (int pa = 0; pa < 2; ++pa)
        for (int pb = 0; pb < 2; ++pb)
          if (!make_map_nhwc_phase(&tmX.m[pa * 2 + pb], x_matrix, a.batch, a.H, a.W, a.C, 2, pa, pb, a.tw, a.th, a.tn))
            return cudaErrorUnknown;
    } else {
      return cudaErrorInvalidValue;
    }
    a.tiles_w = (a.Q + a.tw - 1) / a.tw;
    a.tiles_h = (a.P + a.th - 1) / a.th;
    a.total_kb = a.tiles_w * a.tiles_h * ((a.batch + a.tn - 1) / a.tn);
  } else {
    if (!make_map_2d(&tmDy, dy, a.M, a.dy_ld, a.dy_ld, 64, 64)) return cudaErrorUnknown;
    if (a.mode == kConvGemm) {
      if (!make_map_2d(&tmX.m[0], x_matrix, a.M, a.ncols, a.ncols, 64, 64)) return cudaErrorUnknown;
    } else {
      tmX.m[0] = tmDy;
    }
    for (int i = 1; i < 4; ++i) tmX.m[i] = tmX.m[0];
    a.total_kb = (a.M + 63) / 64;
  }
  if (splits < 1) splits = 1;
  if (splits > a.total_kb) splits = a.total_kb;
  a.kb_per_split = (a.total_kb + splits - 1) / splits;
  splits = (a.total_kb + a.kb_per_split - 1) / a.kb_per_split;
  // one CTA per SM: the deepest ring that fits (the cp.async gather modes need depth > kLag)
  const bool tma_fed = (a.mode == kConvGemm || a.mode == kConvTileFwd || a.mode == kConvStemTma);
  a.stages = kWgMaxStages;
  if (g_force_stages > 0 && g_force_stages <= kWgMaxStages && tma_fed) a.stages = g_force_stages;
  if (a.stages > a.kb_per_split) a.stages = a.kb_per_split;
  if (a.kb_per_split > a.stages && a.stages < (tma_fed ? 2 : kLag + 2)) a.stages = tma_fed ? 2 : kLag + 2;   // see pick_stages
  if (a.stages < 1) a.stages = 1;
  const int smem = wg_smem_bytes(a.stages);
  // narrow outputs (the last 128-channel tile would be at most half full): swap operand roles, 64-channel tiles
  const int co_rem = a.Cout % 128;
  const bool swap = g_wgrad_swap && co_rem > 0 && co_rem <= 64;
  dim3 grid((a.ncols + 127) / 128, swap ? (a.Cout + 63) / 64 : (a.Cout + 127) / 128, splits);
  static bool configured[16] = {};
#define DDL_WG(MODE)                                                                                          \
  do {                                                                                                        \
    auto kern = swap ? conv_wgrad_kernel<MODE, true> : conv_wgrad_kernel<MODE, false>;                        \
    if (!configured[MODE * 2 + (swap ? 1 : 0)]) {                                                             \
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,                 \
                                           wg_smem_bytes(kWgMaxStages));                                      \
      if (e != cudaSuccess) return e;                                                                         \
      configured[MODE * 2 + (swap ? 1 : 0)] = true;                                                           \
    }                                                                                                         \
    kern<<<grid, kThreads, smem, stream>>>(tmDy, tmX, a);                                                     \
  } while (0)
  switch (a.mode) {
    case kConvFwd: DDL_WG(kConvFwd); break;
    case kConvGemm: DDL_WG(kConvGemm); break;
    case kConvStem: DDL_WG(kConvStem); break;
    case kConvTileFwd: DDL_WG(kConvTileFwd); break;
    case kConvStemTma: DDL_WG(kConvStemTma); break;
    default: return cudaErrorInvalidValue;
  }
#undef DDL_WG
  return cudaGetLastError();
}

}  // namespace ddl
