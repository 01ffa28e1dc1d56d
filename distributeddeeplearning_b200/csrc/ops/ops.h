// Host-visible launchers of the memory-bound sm_90a kernels (NHWC bf16 activations).
#pragma once

#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ddl {

struct Fp8Slot {       // one quantised tensor role; lives in a device-resident table (graph replays see live values)
  float amax;          // running max |x| of the current step (cleared by update_scales)
  float scale;         // multiply before the fp8 conversion (power of two)
  float inv_scale;     // 1 / scale: folded into the consuming GEMM's epilogue
  int e5m2;            // 0 = e4m3 (activations, weights), 1 = e5m2 (gradients)
};
struct BnFwdArgs {
  const __nv_bfloat16* x;         // [M][C] conv output
  const __nv_bfloat16* residual;  // optional [M][C]
  __nv_bfloat16* z;               // [M][C]
  const float* sum;               // [C] (train)
  const float* sumsq;             // [C] (train)
  const float* gamma;
  const float* beta;
  float* mean;                    // [C] out (train)
  float* invstd;                  // [C] out (train)
  float* running_mean;            // [C] in/out (may be null in train)
  float* running_var;
  float eps, momentum;
  int M, C, relu;
  uint8_t* mask;                  // optional [M][C/8]: bit i of byte (row, group) = (z[row][8*group + i] > 0).  Written
                                  //   for residual layers so that backward reads 1 bit instead of 16 bits per element
  uint8_t* zq;                    // optional fp8 (e4m3) twin of z for the consuming convolution's tensor-core operand:
  Fp8Slot* zq_slot;               //   z * slot->scale, amax(|z|) folded into the slot (ops/fp8.py: no separate quantise pass)
  int reverse;                    // walk the rows from the END: the producing conv wrote x front to back, so the tail of a
                                  //   tensor larger than L2 is what is still cached (set by the launcher: set_bn_reverse)
};

struct BnBwdArgs {
  const __nv_bfloat16* dz;        // [M][C] gradient wrt z
  const __nv_bfloat16* z;         // [M][C] saved output (ReLU mask)
  const __nv_bfloat16* x;         // [M][C] saved conv output
  __nv_bfloat16* dx;              // [M][C] gradient wrt x
  __nv_bfloat16* dres;            // optional [M][C] gradient wrt residual (= masked dz)
  const float* mean;
  const float* invstd;
  const float* gamma;
  float* dgamma;                  // [C] scratch, zeroed by the caller; receives this call's sums
  float* dbeta;                   // [C] scratch
  float* gamma_grad;              // optional accumulate targets (parameter gradients)
  float* beta_grad;
  const float* beta;              // needed when the ReLU mask is recomputed from x (mask_from_x)
  int M, C, relu;
  int mask_from_x;                // no residual: z > 0  <=>  x*scale + shift > 0, so z is never read
  const uint8_t* zmask;           // residual layers: the bit mask written by the forward kernel (z is never read)
  uint8_t* dxq;                   // optional fp8 (e5m2) twin of dx for the data-gradient convolution that consumes it
  Fp8Slot* dxq_slot;
  int reverse;                    // the REDUCE pass walks the rows from the end (dz was just written front to back; the apply
                                  //   pass then walks forward and finds the rows the reduce pass read last)
};

cudaError_t launch_bn_act_fwd(const BnFwdArgs& a, bool train, int sms, cudaStream_t stream);
// skip_reduce: dgamma / dbeta scratch already hold this layer's sums (fused into the producing dgrad kernel's epilogue)
cudaError_t launch_bn_act_bwd(const BnBwdArgs& a, int sms, cudaStream_t stream, bool skip_reduce = false);

// per-channel sum / sumsq of a bf16 [M][C] tensor (used when the producer had no fused stats)
cudaError_t launch_channel_stats(const __nv_bfloat16* x, float* sum, float* sumsq, int M, int C, int sms,
                                 cudaStream_t stream);

// ---- pooling -------------------------------------------------------------------------------------
struct PoolArgs {
  int N, H, W, C, P, Q, k, stride, pad;
};
// stem fusion (conv -> BN -> ReLU -> max-pool): forward writes only the pooled activation + arg-max codes, backward
// rebuilds BN's input gradient from the pooled gradient (train mode; a.x = raw conv output [N*H*W][C])
cudaError_t launch_bn_relu_maxpool_fwd(const BnFwdArgs& a, const PoolArgs& p, __nv_bfloat16* pooled, uint8_t* argmax,
                                       int sms, cudaStream_t stream);
cudaError_t launch_bn_pool_bwd(const BnBwdArgs& a, const PoolArgs& p, const __nv_bfloat16* dy_pooled, const uint8_t* argmax,
                               int sms, cudaStream_t stream);
cudaError_t launch_maxpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, uint8_t* argmax, const PoolArgs& p,
                               cudaStream_t stream);
cudaError_t launch_maxpool_bwd(const __nv_bfloat16* dy, const uint8_t* argmax, __nv_bfloat16* dx, const PoolArgs& p,
                               cudaStream_t stream);
cudaError_t launch_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, const PoolArgs& p, int count_include_pad,
                               cudaStream_t stream);
cudaError_t launch_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, const PoolArgs& p, int count_include_pad,
                               cudaStream_t stream);
// global average pool: [N][HW][C] -> [N][C] and its backward
cudaError_t launch_global_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int N, int HW, int C,
                                      cudaStream_t stream);
cudaError_t launch_global_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int N, int HW, int C,
                                      cudaStream_t stream);

// ---- loss ----------------------------------------------------------------------------------------
struct XentArgs {
  const __nv_bfloat16* logits;  // [B][ld] (first `classes` columns valid)
  const int64_t* labels;        // [B]
  __nv_bfloat16* dlogits;       // [B][ld] or null ; = (softmax - onehot) * grad_scale, padded cols = 0
  float* loss_sum;              // scalar accumulator: += sum_b loss_b * loss_scale
  float* per_sample;            // optional [B]
  int32_t* correct;             // optional [2]: top-1, top-5 hit counters (+=)
  float loss_scale;             // usually 1/B
  float grad_scale;             // usually 1/B
  int B, classes, ld;
};
cudaError_t launch_softmax_xent(const XentArgs& a, cudaStream_t stream);

// ---- synthetic data ------------------------------------------------------------------------------
// Philox4x32-10 normal(0,1) image batch, NHWC with `cpad` channels (channels >= c_valid are zero)
cudaError_t launch_philox_normal_nhwc(__nv_bfloat16* out, int64_t pixels, int c_valid, int cpad, uint64_t seed,
                                      uint64_t offset, cudaStream_t stream);
cudaError_t launch_philox_labels(int64_t* out, int64_t n, int classes, uint64_t seed, uint64_t offset,
                                 cudaStream_t stream);

// ---- layout / dtype helpers -----------------------------------------------------------------------
// NCHW fp32 -> NHWC(cpad) bf16 with per-channel (x - mean) / std   (real-image input path, K21)
cudaError_t launch_nchw_to_nhwc_norm(const float* in, __nv_bfloat16* out, int N, int C, int H, int W, int cpad,
                                     const float* mean, const float* stdv, cudaStream_t stream);
// uint8 NHWC3 -> bf16 NHWC4 with (x/255 - mean)/std  (end-to-end input path: 3 bytes/pixel over PCIe)
cudaError_t launch_nhwc_u8_to_nhwc4(const uint8_t* in, __nv_bfloat16* out, int64_t pixels, const float* mean,
                                    const float* stdv, cudaStream_t stream);
cudaError_t launch_cast_f32_bf16(const float* in, __nv_bfloat16* out, int64_t n, cudaStream_t stream);
// stem weights: fp32 [Cout][R][S][Cin<=4] (KRSC) <-> packed bf16 [Cout][KBR][SP][4] (zero padded)
cudaError_t launch_pack_stem_weight(const float* w, __nv_bfloat16* packed, int Cout, int R, int S, int Cin, int RP,
                                    int SP, cudaStream_t stream);
cudaError_t launch_unpack_stem_grad(const float* packed, float* gw, int Cout, int R, int S, int Cin, int RP, int SP,
                                    cudaStream_t stream);

// ---- bias / activation / dropout (VGG / AlexNet classifier paths) ---------------------------------
// dy_masked = dy * (z > 0) ; dbias[c] += sum_m dy_masked    (z = relu(conv + bias) saved output)
cudaError_t launch_bias_relu_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* z, __nv_bfloat16* dx, float* dbias,
                                 int M, int C, int c_valid, int relu, int sms, cudaStream_t stream);
cudaError_t launch_dropout(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, float p, uint64_t seed,
                           uint64_t offset, const int64_t* step, cudaStream_t stream);
// y = a + b (bf16)
// NHWC4 image [N][H][W] (8-byte pixels) -> zero-bordered, G-row-interleaved [N][Hp][Wp][G][4] with the source at
// (pt, pl): position (h, w) holds the pixels of rows h .. h+G-1.  Operand layout of the TMA-fed stem convolution
// (conv_gemm.cuh kConvStemTma): SP taps x G rows x 4 channels of one output pixel are 128 contiguous bytes.
cudaError_t launch_pad_nhwc4(const __nv_bfloat16* in, __nv_bfloat16* out, int N, int H, int W, int Hp, int Wp, int pt,
                             int pl, int G, cudaStream_t stream);
// Channel concatenation of up to kCatMax NHWC tensors (Inception / DenseNet, SURVEY.md K20): gather = parts -> whole,
// scatter (backward) = whole -> parts.  Every part's channel count is a multiple of 8.
constexpr int kCatMax = 8;
struct CatArgs {
  __nv_bfloat16* part[kCatMax];
  int c[kCatMax];          // channels of each part
  int n;                   // parts
  __nv_bfloat16* whole;    // [M][ctot]
  int M, ctot;
};
cudaError_t launch_concat_channels(const CatArgs& a, bool scatter, cudaStream_t stream);
cudaError_t launch_add_bf16(const __nv_bfloat16* a, const __nv_bfloat16* b, __nv_bfloat16* y, int64_t n,
                            cudaStream_t stream);

// ---- FP8 operand preparation (fp8.cu) ----------------------------------------------------------------
cudaError_t launch_fp8_quantize(const __nv_bfloat16* x, uint8_t* out, int64_t n, Fp8Slot* slot, bool e5m2, int sms,
                                cudaStream_t stream);
cudaError_t launch_fp8_amax(const __nv_bfloat16* x, int64_t n, Fp8Slot* slot, int sms, cudaStream_t stream);
cudaError_t launch_fp8_update_scales(Fp8Slot* slots, int n, cudaStream_t stream);
// codes [rows][taps][cols] -> [cols][taps][rows] (the data gradient's K-major copy of quantised weights)
cudaError_t launch_fp8_transpose_taps(const uint8_t* in, uint8_t* out, int rows, int taps, int cols, cudaStream_t stream);
// MX (OCP microscaling) quantisation of a row-major bf16 matrix [rows][K], K % 128 == 0: e4m3 codes + one UE8M0 scale per
// 32 consecutive K elements of a row, written in 512-byte atoms (ConvArgs::sfa): sf must hold
// ceil(rows/128) * (K/128) * 512 bytes and be zero-initialised (rows beyond `rows` keep scale byte 0).
cudaError_t launch_fp8_quantize_mx(const __nv_bfloat16* x, uint8_t* out, uint8_t* sf, int64_t rows, int64_t K, int sms,
                                   cudaStream_t stream);

}  // namespace ddl
