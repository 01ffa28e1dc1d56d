// FP8 (e4m3 / e5m2) operand preparation for the fp8 wgmma conv / GEMM path (BASELINE config #3:
// ResNet-50 with 8-bit tensor-core operands; the reference's only reduced-precision switch is the TF benchmark's
// `--use_fp16`, TensorFlow_benchmark/tensorflow_benchmark.py:51,77).
//
// Recipe (delayed per-tensor scaling, the recipe FP8 training stacks converged on):
//   * every quantised tensor role (a layer's input activation, its weight matrix, its output gradient) owns one slot
//     {amax, scale, inv_scale, calibrated} in a device-resident table;
//   * `quantize` multiplies by the slot's CURRENT scale, saturates to the format's finite range and, in the same
//     pass, folds |x| into the slot's amax (atomicMax on the bit pattern: non-negative floats order like integers);
//   * once per step `update_scales` turns every amax into next step's power-of-two scale (so scaling itself is exact)
//     and clears it — ONE launch for the whole model, captured into the step's CUDA graph like everything else;
//   * a slot's first use is calibrated with a separate amax pass so that step 0 is not quantised blindly.
// The GEMM epilogue multiplies the fp32 accumulator by inv_scale(A) * inv_scale(B) (read from the table), so
// everything downstream (BN statistics, bf16 outputs, wgrad, optimizer) is unchanged.
#include "../common.cuh"
#include "ops.h"

#include <cuda_fp8.h>

namespace ddl {

namespace {

constexpr float kE4m3Max = 448.f;
constexpr float kE5m2Max = 57344.f;

DDL_DEVICE float block_max(float v) {
  __shared__ float s[32];
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x < 32) {
    float w = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0.f;
    w = warp_max(w);
    if (threadIdx.x == 0) s[0] = w;
  }
  __syncthreads();
  return s[0];
}

// out[i] = fp8(x[i] * scale);  slot->amax = max(slot->amax, max |x|)
template <bool E5M2>
__global__ void __launch_bounds__(256) quantize_fp8_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ out,
                                                           int64_t n8, Fp8Slot* slot) {
  const float scale = slot->scale;
  float amax = 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const uint4 v = ld_stream_u4(reinterpret_cast<const uint4*>(x) + i);
    const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(d.x), fabsf(d.y))));
    uint2 o;
    o.x = fp8_cvt4<E5M2>(a.x * scale, a.y * scale, b.x * scale, b.y * scale);
    o.y = fp8_cvt4<E5M2>(c.x * scale, c.y * scale, d.x * scale, d.y * scale);
    reinterpret_cast<uint2*>(out)[i] = o;
  }
  amax = block_max(amax);
  if (threadIdx.x == 0 && amax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(&slot->amax), __float_as_uint(amax));
}

__global__ void __launch_bounds__(256) amax_bf16_kernel(const __nv_bfloat16* __restrict__ x, int64_t n8, Fp8Slot* slot) {
  float amax = 0.f;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n8; i += stride) {
    const uint4 v = ld_stream_u4(reinterpret_cast<const uint4*>(x) + i);
    const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))));
    amax = fmaxf(amax, fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(d.x), fabsf(d.y))));
  }
  amax = block_max(amax);
  if (threadIdx.x == 0 && amax > 0.f) atomicMax(reinterpret_cast<unsigned int*>(&slot->amax), __float_as_uint(amax));
}

// scale = 2^floor(log2(fmax / (amax * margin))): a power of two, so x * scale only shifts the exponent
DDL_DEVICE void slot_update(Fp8Slot& s) {
  const float amax = s.amax;
  if (amax > 0.f && isfinite(amax)) {
    const float fmax = s.e5m2 ? kE5m2Max : kE4m3Max;
    int e;
    frexpf(fmax / (amax * 1.0f), &e);           // fmax/amax = m * 2^e, m in [0.5, 1)  ->  2^(e-1) <= fmax/amax
    float sc = ldexpf(1.0f, e - 1);
    sc = fminf(fmaxf(sc, 1.0f / 16777216.f), 16777216.f * 4096.f);
    s.scale = sc;
    s.inv_scale = 1.0f / sc;
  }
  s.amax = 0.f;                                  // tensors that were not touched this step keep their scale
}

__global__ void update_scales_kernel(Fp8Slot* slots, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) slot_update(slots[i]);
}

// MX quantisation: thread = 8 consecutive K elements; the 4 threads of a 32-element block agree on the block's amax
// with two shuffles.  scale = 2^e with e = ceil(log2(amax / 448)) (so amax / scale <= 448), stored as UE8M0 (e + 127).
__global__ void __launch_bounds__(256) quantize_mx_kernel(const __nv_bfloat16* __restrict__ x, uint8_t* __restrict__ out,
                                                          uint8_t* __restrict__ sf, int64_t rows, int64_t K) {
  const int64_t vec_per_row = K / 8;
  const int64_t total = rows * vec_per_row;
  const int64_t kb128 = K / 128;
  // the bound is a multiple of the warp size (as are the start and the stride): a warp is in the loop as a whole, which
  // the full-mask shuffles below require
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < ((total + 31) / 32) * 32;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const bool live = i < total;
    uint4 v = make_uint4(0, 0, 0, 0);
    if (live) v = ld_stream_u4(reinterpret_cast<const uint4*>(x) + i);
    const float2 a = unpack_bf16x2(v.x), b = unpack_bf16x2(v.y), c = unpack_bf16x2(v.z), d = unpack_bf16x2(v.w);
    float amax = fmaxf(fmaxf(fmaxf(fabsf(a.x), fabsf(a.y)), fmaxf(fabsf(b.x), fabsf(b.y))),
                       fmaxf(fmaxf(fabsf(c.x), fabsf(c.y)), fmaxf(fabsf(d.x), fabsf(d.y))));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
    int e = 0;
    if (amax > 0.f) {
      int ex;
      const float m = frexpf(amax / kE4m3Max, &ex);          // amax/448 = m * 2^ex, m in [0.5, 1)
      e = (m == 0.5f) ? ex - 1 : ex;                          // smallest e with amax / 2^e <= 448
      e = max(-127, min(127, e));
    }
    const float inv = ldexpf(1.0f, -e);
    if (live) {
      uint2 o;
      o.x = fp8_cvt4<false>(a.x * inv, a.y * inv, b.x * inv, b.y * inv);
      o.y = fp8_cvt4<false>(c.x * inv, c.y * inv, d.x * inv, d.y * inv);
      reinterpret_cast<uint2*>(out)[i] = o;
      if ((i & 3) == 0) {                                     // first thread of the 32-element block writes its scale
        const int64_t row = i / vec_per_row;
        const int64_t k32 = (i - row * vec_per_row) / 4;      // 32-element block index along K
        const int64_t r = row & 127;
        sf[((row >> 7) * kb128 + (k32 >> 2)) * 512 + (r & 31) * 16 + (r >> 5) * 4 + (k32 & 3)] =
            static_cast<uint8_t>(e + 127);
      }
    }
  }
}

}  // namespace

cudaError_t launch_fp8_quantize_mx(const __nv_bfloat16* x, uint8_t* out, uint8_t* sf, int64_t rows, int64_t K, int sms,
                                   cudaStream_t stream) {
  if (K % 128 != 0 || rows <= 0) return cudaErrorInvalidValue;
  const int64_t total = rows * (K / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 8LL * sms) blocks = 8LL * sms;
  quantize_mx_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, out, sf, rows, K);
  return cudaGetLastError();
}

// fp8 codes [rows][taps][cols] -> [cols][taps][rows]: the data gradient's K-major copy of a quantised weight matrix.
// 32 x 32 byte tiles through shared memory (coalesced reads and writes), one grid z slice per filter tap.
__global__ void transpose_taps_u8_kernel(const uint8_t* __restrict__ in, uint8_t* __restrict__ out, int rows, int taps,
                                         int cols) {
  __shared__ uint8_t t[32][33];
  const int tap = blockIdx.z;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int r = r0 + i, c = c0 + threadIdx.x;
    if (r < rows && c < cols) t[i][threadIdx.x] = in[(static_cast<size_t>(r) * taps + tap) * cols + c];
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, r = r0 + threadIdx.x;
    if (c < cols && r < rows) out[(static_cast<size_t>(c) * taps + tap) * rows + r] = t[threadIdx.x][i];
  }
}

cudaError_t launch_fp8_transpose_taps(const uint8_t* in, uint8_t* out, int rows, int taps, int cols, cudaStream_t stream) {
  if (rows <= 0 || taps <= 0 || cols <= 0 || taps > 65535) return cudaErrorInvalidValue;
  const dim3 grid((cols + 31) / 32, (rows + 31) / 32, taps);
  transpose_taps_u8_kernel<<<grid, dim3(32, 8), 0, stream>>>(in, out, rows, taps, cols);
  return cudaGetLastError();
}

cudaError_t launch_fp8_quantize(const __nv_bfloat16* x, uint8_t* out, int64_t n, Fp8Slot* slot, bool e5m2, int sms,
                                cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  const int64_t n8 = n / 8;
  int64_t blocks = (n8 + 255) / 256;
  if (blocks > 8LL * sms) blocks = 8LL * sms;
  if (blocks < 1) blocks = 1;
  if (e5m2) quantize_fp8_kernel<true><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, out, n8, slot);
  else quantize_fp8_kernel<false><<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, out, n8, slot);
  return cudaGetLastError();
}

cudaError_t launch_fp8_amax(const __nv_bfloat16* x, int64_t n, Fp8Slot* slot, int sms, cudaStream_t stream) {
  if (n % 8 != 0) return cudaErrorInvalidValue;
  const int64_t n8 = n / 8;
  int64_t blocks = (n8 + 255) / 256;
  if (blocks > 8LL * sms) blocks = 8LL * sms;
  if (blocks < 1) blocks = 1;
  amax_bf16_kernel<<<static_cast<unsigned>(blocks), 256, 0, stream>>>(x, n8, slot);
  return cudaGetLastError();
}

cudaError_t launch_fp8_update_scales(Fp8Slot* slots, int n, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  update_scales_kernel<<<(n + 127) / 128, 128, 0, stream>>>(slots, n);
  return cudaGetLastError();
}

}  // namespace ddl
