// Shared device helpers for the b200-ddl kernels (sm_90a).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#define DDL_DEVICE __device__ __forceinline__

namespace ddl {

constexpr int kMaxWorld = 8;
constexpr int kWarp = 32;

// ---------------------------------------------------------------------------------------------
// programmatic dependent launch (PDL): a kernel launched with launch_pdl() (launch.h) may become resident while its
// predecessor in the stream is still draining; everything it does before pdl_wait() (index math, barrier init,
// tensor-map prefetch) overlaps that tail.  RULE: pdl_wait() comes before the first access to global
// memory — it returns once the predecessor grid has completed and its writes are visible (no-op without the launch
// attribute).  pdl_trigger() lets the NEXT kernel in the stream start its own preamble early.
// ---------------------------------------------------------------------------------------------
// Triggering is a mode per translation unit (c_pdl_trigger, set_pdl): 0 plain stream order, 1 (default) the launch
// attribute only (dependents launch as the last blocks exit), 2 the conv kernels trigger at their last tile, 3 every
// block triggers at its start.  Every kernel here assigns its tiles / rows statically to a grid sized for an even spread,
// so dependents that become resident early land unevenly on the SMs; the default was chosen on that ground and was not
// re-measured on H100.
__constant__ int c_pdl_trigger;       // 0 = never explicitly, 1 = at the last tile (conv), 2 = at block start
DDL_DEVICE void pdl_trigger() {
  if (c_pdl_trigger == 2) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
DDL_DEVICE void pdl_trigger_last_tile() {
  if (c_pdl_trigger == 1) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
DDL_DEVICE void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ---------------------------------------------------------------------------------------------
// small numeric helpers
// ---------------------------------------------------------------------------------------------
DDL_DEVICE uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
DDL_DEVICE float2 unpack_bf16x2(uint32_t v) {
  __nv_bfloat162 b = *reinterpret_cast<__nv_bfloat162*>(&v);
  return __bfloat1622float2(b);
}
DDL_DEVICE float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

DDL_DEVICE float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
DDL_DEVICE float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// four floats -> four fp8 codes (e4m3 or e5m2, round-to-nearest, saturating to the finite range), a at the lowest byte
template <bool E5M2>
DDL_DEVICE uint32_t fp8_cvt4(float a, float b, float c, float d) {
  uint16_t lo, hi;
  if (E5M2) {
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  } else {
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  }
  return static_cast<uint32_t>(lo) | (static_cast<uint32_t>(hi) << 16);
}

// 16-byte global accesses with cache hints (streaming data: do not pollute L1)
DDL_DEVICE uint4 ld_stream_u4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
DDL_DEVICE uint2 ld_stream_u2(const void* p) {
  uint2 r;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
  return r;
}
DDL_DEVICE void st_stream_u4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};"
               :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}
DDL_DEVICE void st_stream_u2(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" :: "l"(p), "r"(v.x), "r"(v.y) : "memory");
}

DDL_DEVICE uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------------------------------------
// Philox4x32-10 counter-based RNG (Salmon et al.), one 128-bit block per call
// ---------------------------------------------------------------------------------------------
DDL_DEVICE uint4 philox4x32_10(uint4 ctr, uint2 key) {
  constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}
// uniform in (0,1]
DDL_DEVICE float u32_to_unit(uint32_t x) { return (static_cast<float>(x >> 8) + 1.0f) * (1.0f / 16777216.0f); }
// Box-Muller: two standard normals from two uint32
DDL_DEVICE float2 box_muller(uint32_t a, uint32_t b) {
  float u1 = u32_to_unit(a), u2 = u32_to_unit(b);
  float r = sqrtf(-2.0f * __logf(u1));
  float s, c;
  __sincosf(6.283185307179586f * u2, &s, &c);
  return make_float2(r * c, r * s);
}

}  // namespace ddl
