// Device-side image augmentation of the ImageNet trainers (data/images.py, augment="device"): the resized crop, the
// horizontal flip and the normalisation of a batch of ragged uint8 regions, written as the bf16 NHWC4 activations the
// stems read.
//
// Input: one packed uint8 buffer holding B regions, each HWC3 at its own byte offset, and a float64 descriptor per image
// [offset, Hr, Wr, sy, sx, oy, ox, flip].  Each axis is resampled with the antialiased bilinear (triangle) filter of
// torch's interpolate(antialias=True) and of PIL's BILINEAR resample; for region length L, scale s, offset o and output
// index i:
//   center = s (i + o + 0.5),  support = max(s, 1),  inv = s >= 1 ? 1 / s : 1
//   taps j in [max(int(center - support + 0.5), 0), min(int(center + support + 0.5), L)),
//   w_j = max(0, 1 - |(j - center + 0.5) inv|), normalised by their sum.
// The taps clamp to the region.  A train crop is the region itself (s = crop / S, o = 0); a validation image is the
// whole decoded image (s = orig / resized, o = the centre crop's offset).  Output: (v / 255 - mean) / std, channel 3 = 0;
// the flip mirrors the output column index.
//
// Mapping: a CTA owns one image, a band of kRcRows output rows and kRcCols output columns, one column per thread.  It
// streams the input rows the band's vertical taps cover: each thread filters its column's horizontal taps of the row
// into three fp32 sums, then adds them with the row's vertical weight into the band's fp32 accumulators, which live in
// registers.  Shared memory holds only the band's vertical tap tables, so it is bounded whatever the scale; any
// downscale factor and upscaling take the same path.  No atomics: every output pixel is summed by one thread in a fixed
// order.  Each thread stores its pixels as 8-byte NHWC4 words, so a warp's stores are one contiguous 256-byte row run.
#include "../common.cuh"
#include "ops.h"
#include "../launch.h"

namespace ddl {

namespace {

constexpr int kRcCols = 128;   // output columns per CTA (one per thread)
constexpr int kRcRows = 8;     // output rows per CTA

// the taps of output index i on one axis: first tap lo, count n, center - lo, 1 / support scale and 1 / weight sum
DDL_DEVICE void rc_axis(double s, double o, int i, int L, int& lo, int& n, float& frac, float& inv, float& norm) {
  const double center = s * (i + o + 0.5);
  const double support = s >= 1.0 ? s : 1.0;
  inv = s >= 1.0 ? static_cast<float>(1.0 / s) : 1.f;
  lo = max(static_cast<int>(center - support + 0.5), 0);            // int() truncates, like the reference formula
  n = min(static_cast<int>(center + support + 0.5), L) - lo;
  frac = static_cast<float>(center - lo);
  float sum = 0.f;
  for (int t = 0; t < n; ++t) sum += fmaxf(0.f, 1.f - fabsf((t + 0.5f - frac) * inv));
  norm = sum > 0.f ? 1.f / sum : 0.f;
}

__global__ void __launch_bounds__(kRcCols) resized_crop_kernel(const uint8_t* __restrict__ src,
                                                               const double* __restrict__ desc,
                                                               __nv_bfloat16* __restrict__ out, int S,
                                                               const float* __restrict__ mean,
                                                               const float* __restrict__ stdv) {
  __shared__ int s_lo[kRcRows], s_n[kRcRows];
  __shared__ float s_frac[kRcRows], s_w[kRcRows];
  pdl_trigger();
  pdl_wait();
  const double* d = desc + static_cast<int64_t>(blockIdx.z) * 8;
  const int64_t off = static_cast<int64_t>(d[0]);
  const int Hr = static_cast<int>(d[1]), Wr = static_cast<int>(d[2]);
  const double sy = d[3], sx = d[4];
  const int y0 = blockIdx.y * kRcRows;
  const float invy = sy >= 1.0 ? static_cast<float>(1.0 / sy) : 1.f;
  if (threadIdx.x < kRcRows) {
    int lo = 0, n = 0;                 // rows past the image's last output row take no taps
    float frac = 0.f, inv, norm = 0.f;
    if (y0 + static_cast<int>(threadIdx.x) < S) rc_axis(sy, d[5], y0 + threadIdx.x, Hr, lo, n, frac, inv, norm);
    s_lo[threadIdx.x] = lo;
    s_n[threadIdx.x] = n;
    s_frac[threadIdx.x] = frac;
    s_w[threadIdx.x] = norm;
  }
  __syncthreads();
  const int xo = blockIdx.x * kRcCols + threadIdx.x;
  if (xo >= S) return;
  int lx, nx;
  float fx, ix, wx;
  rc_axis(sx, d[6], d[7] != 0.0 ? S - 1 - xo : xo, Wr, lx, nx, fx, ix, wx);
  // vertical taps are monotone in the output row: the band reads rows [lo of its first row, hi of its last row)
  const int rows = min(kRcRows, S - y0);
  const int r0 = s_lo[0], r1 = s_lo[rows - 1] + s_n[rows - 1];
  float acc[kRcRows][3];
#pragma unroll
  for (int k = 0; k < kRcRows; ++k) acc[k][0] = acc[k][1] = acc[k][2] = 0.f;
  const uint8_t* col = src + off + static_cast<int64_t>(lx) * 3;
  for (int r = r0; r < r1; ++r) {
    const uint8_t* p = col + static_cast<int64_t>(r) * Wr * 3;
    float h0 = 0.f, h1 = 0.f, h2 = 0.f;
    for (int t = 0; t < nx; ++t, p += 3) {
      const float w = fmaxf(0.f, 1.f - fabsf((t + 0.5f - fx) * ix));
      h0 = fmaf(w, static_cast<float>(__ldg(p)), h0);
      h1 = fmaf(w, static_cast<float>(__ldg(p + 1)), h1);
      h2 = fmaf(w, static_cast<float>(__ldg(p + 2)), h2);
    }
#pragma unroll
    for (int k = 0; k < kRcRows; ++k) {
      const int t = r - s_lo[k];
      if (t >= 0 && t < s_n[k]) {
        const float w = fmaxf(0.f, 1.f - fabsf((t + 0.5f - s_frac[k]) * invy)) * s_w[k];
        acc[k][0] = fmaf(w, h0, acc[k][0]);
        acc[k][1] = fmaf(w, h1, acc[k][1]);
        acc[k][2] = fmaf(w, h2, acc[k][2]);
      }
    }
  }
  const float m0 = mean[0], m1 = mean[1], m2 = mean[2];
  const float is0 = 1.f / stdv[0], is1 = 1.f / stdv[1], is2 = 1.f / stdv[2];
  const float sc = wx / 255.f;
  uint2* o = reinterpret_cast<uint2*>(out) + (static_cast<int64_t>(blockIdx.z) * S + y0) * S + xo;
#pragma unroll
  for (int k = 0; k < kRcRows; ++k) {
    if (k < rows) {
      const float c0 = (acc[k][0] * sc - m0) * is0, c1 = (acc[k][1] * sc - m1) * is1, c2 = (acc[k][2] * sc - m2) * is2;
      o[static_cast<int64_t>(k) * S] = make_uint2(pack_bf16x2(c0, c1), pack_bf16x2(c2, 0.f));
    }
  }
}

}  // namespace

cudaError_t launch_resized_crop(const uint8_t* src, const double* desc, __nv_bfloat16* out, int B, int S,
                                const float* mean, const float* stdv, cudaStream_t stream) {
  if (B <= 0 || S <= 0) return cudaSuccess;
  const dim3 grid((S + kRcCols - 1) / kRcCols, (S + kRcRows - 1) / kRcRows, B);
  return launch_pdl(resized_crop_kernel, grid, dim3(kRcCols), 0, stream, 1, src, desc, out, S, mean, stdv);
}

}  // namespace ddl
