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
  const float* sample_scale;      // optional [M / hw] per-sample scale of the BN output before the residual add
  int hw;                         //   (stochastic depth: z = BN(x) * sample_scale[row / hw] + residual; no activation,
                                  //   or relu == 6: z = silu(BN(x)) * sample_scale[row / hw] + residual)
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
  const float* sample_scale;      // optional, as in BnFwdArgs: BN sees dz * sample_scale[row / hw], dres = dz
  int hw;                         //   (relu == 6: the SiLU's input sees dz * sample_scale[row / hw] * silu'(v))
};

cudaError_t launch_bn_act_fwd(const BnFwdArgs& a, bool train, int sms, cudaStream_t stream);
// skip_reduce: dgamma / dbeta scratch already hold this layer's sums (fused into the producing dgrad kernel's epilogue)
cudaError_t launch_bn_act_bwd(const BnBwdArgs& a, int sms, cudaStream_t stream, bool skip_reduce = false);

// per-channel sum / sumsq of a bf16 [M][C] tensor (used when the producer had no fused stats)
cudaError_t launch_channel_stats(const __nv_bfloat16* x, float* sum, float* sumsq, int M, int C, int sms,
                                 cudaStream_t stream);

// ---- depthwise convolution (depthwise.cu: 3x3, depthwise5.cu: 5x5) ----------------------------------------
// groups == Cin == Cout = C (C % 8 == 0), k x k with k = 3 (padding 1) or 5 (padding 2), stride 1 or 2;
// x [N][H][W][C], y / dy [N][P][Q][C] bf16
struct DwConvArgs {
  const __nv_bfloat16* x;         // forward / wgrad input
  const __nv_bfloat16* dy;        // dgrad / wgrad output gradient
  const __nv_bfloat16* w;         // [C][k][k] bf16
  __nv_bfloat16* y;               // forward: y;  dgrad: dx [N][H][W][C]
  float* sum;                     // forward, optional: per-channel sum / sum of squares of the bf16 y (+=, zeroed
  float* sumsq;                   //   by the caller)
  float* gw;                      // wgrad: fp32 [C][k][k] gradient, accumulated (+=)
  int N, H, W, C, P, Q, stride;
  int lg_gpc;                     // set by the launcher: log2 of the 8-channel groups per block
};
cudaError_t launch_dwconv_fwd(const DwConvArgs& a, int sms, cudaStream_t stream);
cudaError_t launch_dwconv_dgrad(const DwConvArgs& a, int sms, cudaStream_t stream);
cudaError_t launch_dwconv_wgrad(const DwConvArgs& a, int sms, cudaStream_t stream);
cudaError_t launch_dwconv5_fwd(const DwConvArgs& a, int sms, cudaStream_t stream);
cudaError_t launch_dwconv5_dgrad(const DwConvArgs& a, int sms, cudaStream_t stream);
cudaError_t launch_dwconv5_wgrad(const DwConvArgs& a, int sms, cudaStream_t stream);
// ---- depthwise 7x7 with a bias (depthwise7.cu; ConvNeXt): stride 1, padding 3, x / y / dy / dx [N][H][W][C] bf16 ----
struct Dw7Args {
  const __nv_bfloat16* x;         // forward / wgrad input
  const __nv_bfloat16* dy;        // dgrad / wgrad output gradient
  const __nv_bfloat16* w;         // [C][7][7] bf16
  const float* bias;              // forward: fp32 [C]
  const __nv_bfloat16* add;       // dgrad, optional: added to dx in its store (the block's residual gradient)
  __nv_bfloat16* y;               // forward: y;  dgrad: dx
  float* gw;                      // wgrad: fp32 [C][7][7] gradient, accumulated (+=)
  float* gb;                      // wgrad, optional: fp32 [C] bias gradient, accumulated (+=)
  int N, H, W, C;
  int lg_gpc;                     // set by the launcher: log2 of the 8-channel groups per block
};
// l1: the L1 mapping of the 5x5 kernels instead of the shared-memory halo tile (for timing the two against each other)
cudaError_t launch_dwconv7_fwd(const Dw7Args& a, int sms, bool l1, cudaStream_t stream);
cudaError_t launch_dwconv7_dgrad(const Dw7Args& a, int sms, bool l1, cudaStream_t stream);
cudaError_t launch_dwconv7_wgrad(const Dw7Args& a, int sms, cudaStream_t stream);

// ---- ConvNeXt row kernels (convnext.cu) ------------------------------------------------------------------------------
// LayerNorm over the C channels of each row of a bf16 [M][C] matrix (an NHWC activation or [N][C]), C % 8 == 0 and
// C / 8 = T * V with T a power of two <= 32 threads per row and V <= 6 vectors per thread.
// forward: y = (x - mean) * rstd * gamma + beta, saving fp32 mean / rstd [M]
cudaError_t launch_layer_norm_fwd(const __nv_bfloat16* x, const float* gamma, const float* beta, __nv_bfloat16* y,
                                  float* mean, float* rstd, int M, int C, float eps, int sms, cudaStream_t stream);
// backward: dx = rstd * (g dy - mean_c(g dy) - xhat * mean_c(g dy xhat)), g = gamma; dgamma += sum_m dy xhat,
// dbeta += sum_m dy (each optional)
cudaError_t launch_layer_norm_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean, const float* rstd,
                                  const float* gamma, __nv_bfloat16* dx, float* dgamma, float* dbeta, int M, int C, int sms,
                                  cudaStream_t stream);
// exact GELU on n bf16 elements (n % 8 == 0): g = h * Phi(h)
cudaError_t launch_gelu_fwd(const __nv_bfloat16* h, __nv_bfloat16* g, int64_t n, int sms, cudaStream_t stream);
// dh = dg * (Phi(h) + h * phi(h)) on [M][C]; dbias[c] += sum_m dh (optional): fc1's bias gradient, summed over the
// stored bf16 dh (as bias_relu_bwd sums its bf16 dy)
cudaError_t launch_gelu_bwd(const __nv_bfloat16* dg, const __nv_bfloat16* h, __nv_bfloat16* dh, float* dbias, int M, int C,
                            int sms, cudaStream_t stream);
// layer scale + stochastic depth + residual on [M][C] (M = N * hw): z = ls[c] * y * keep[m / hw] + x (keep optional)
cudaError_t launch_layer_scale_fwd(const __nv_bfloat16* y, const float* ls, const float* keep, const __nv_bfloat16* x,
                                   __nv_bfloat16* z, int M, int C, int hw, int sms, cudaStream_t stream);
// dy = dz * ls[c] * keep[m / hw];  dls[c] += sum_m dz * keep * y;  dbias[c] += sum_m dy over the stored bf16 dy
// (dls / dbias optional)
cudaError_t launch_layer_scale_bwd(const __nv_bfloat16* dz, const __nv_bfloat16* y, const float* ls, const float* keep,
                                   __nv_bfloat16* dy, float* dls, float* dbias, int M, int C, int hw, int sms,
                                   cudaStream_t stream);

// ---- multi-head self-attention, head dim 64 (attention.cu; ViT) -------------------------------------------------------
// qkv [N*L][3C] bf16 (head h: Q, K, V at columns 64h, C + 64h, 2C + 64h), C = 64 H.  forward: o [N*L][C] =
// softmax(Q K^T / 8) V per (image, head), lse [N][H][L] fp32 natural-log log-sum-exp of the scaled scores.
cudaError_t launch_attention_fwd(const __nv_bfloat16* qkv, __nv_bfloat16* o, float* lse, int N, int L, int H, int C,
                                 cudaStream_t stream);
// backward (two kernels): dqkv [N*L][3C] in qkv's layout from dout [N*L][C] and the saved qkv, o, lse; delta [N][H][L]
// fp32 receives D = rowsum(dout o o)
cudaError_t launch_attention_bwd(const __nv_bfloat16* qkv, const __nv_bfloat16* o, const __nv_bfloat16* dout,
                                 const float* lse, float* delta, __nv_bfloat16* dqkv, int N, int L, int H, int C,
                                 cudaStream_t stream);

// ---- ViT row kernels (vit.cu) ------------------------------------------------------------------------------------------
// x1 = x + add, y = LayerNorm(x1) on [M][C] rows (the LayerNorm mapping of convnext.cu), saving fp32 mean / rstd [M]
cudaError_t launch_add_layer_norm_fwd(const __nv_bfloat16* x, const __nv_bfloat16* add, const float* gamma,
                                      const float* beta, __nv_bfloat16* x1, __nv_bfloat16* y, float* mean, float* rstd,
                                      int M, int C, float eps, int sms, cudaStream_t stream);
// dx = LayerNorm_bwd(dy) + dres; dgamma / dbeta as launch_layer_norm_bwd (optional)
cudaError_t launch_layer_norm_bwd_add(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean,
                                      const float* rstd, const float* gamma, const __nv_bfloat16* dres, __nv_bfloat16* dx,
                                      float* dgamma, float* dbeta, int M, int C, int sms, cudaStream_t stream);
// NHWC4 image [N][H][W][4] -> patch rows [N * (H/P) * (W/P)][P*P*3] in (r, s, c) order
cudaError_t launch_patchify(const __nv_bfloat16* img, __nv_bfloat16* out, int N, int H, int W, int P, int sms,
                            cudaStream_t stream);
// tok [N*L][C] = (cls | patch [N*(L-1)][C]) + pos [L][C]  (cls, pos fp32)
cudaError_t launch_tokens_fwd(const __nv_bfloat16* patch, const float* cls, const float* pos, __nv_bfloat16* tok, int N,
                              int L, int C, int sms, cudaStream_t stream);
// dpatch = rows 1.. of every image of dtok (optional); colsum [L][C] fp32 scratch; dpos[l] += sum_n dtok[n, l],
// dcls += sum_n dtok[n, 0], dbias += sum_{n, l >= 1} dtok[n, l] (each optional), in a fixed order (two kernels)
cudaError_t launch_tokens_bwd(const __nv_bfloat16* dtok, __nv_bfloat16* dpatch, float* colsum, float* dpos, float* dcls,
                              float* dbias, int N, int L, int C, cudaStream_t stream);

// ---- Swin: shifted-window attention, window 7, head dim 32 (window_attention.cu) ---------------------------------------
// qkv [N*H*W][3C] bf16 in image order (head h: Q, K, V at columns 32h, C + 32h, 2C + 32h), C = 32 heads, H and W
// multiples of 7, shift (sy, sx) in [0, 7) (0 on a side of 7).  forward: o [N*H*W][C] and lse [N*H*W][heads] fp32 of the
// windows of the map rolled by -shift, with the relative-position bias table [169][heads] fp32 and the shifted-window mask.
cudaError_t launch_window_attention_fwd(const __nv_bfloat16* qkv, const float* table, __nv_bfloat16* o, float* lse,
                                        int N, int H, int W, int heads, int C, int sy, int sx, cudaStream_t stream);
// backward (three kernels, deterministic): dqkv [N*H*W][3C] in qkv's layout; dtable [169][heads] += the bias gradient
// (optional); scratch holds window_attention_bwd_scratch_floats(N, H, heads) fp32
cudaError_t launch_window_attention_bwd(const __nv_bfloat16* qkv, const float* table, const __nv_bfloat16* o,
                                        const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv, float* dtable,
                                        float* scratch, int N, int H, int W, int heads, int C, int sy, int sx,
                                        cudaStream_t stream);
size_t window_attention_bwd_scratch_floats(int N, int H, int heads);

// ---- MaxViT: partition attention, 7 x 7 partitions, head dim 32 (window_attention.cu) --------------------------------
// qkv [N*H*W][3C] bf16 in image order (head h: Q, K, V at columns 32h, C + 32h, 2C + 32h), C = 32 heads, H = W a multiple
// of 7.  grid: the 49 tokens of sequence (i, j) sit at pixels (a H/7 + i, b H/7 + j); else (the window partition) at
// (7i + a, 7j + b).  forward: o [N*H*W][C] and lse [N*H*W][heads] fp32 with logits q . k * scale + table[169][heads].
cudaError_t launch_grid_attention_fwd(const __nv_bfloat16* qkv, const float* table, __nv_bfloat16* o, float* lse,
                                      int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream);
// backward (three kernels, deterministic): dqkv [N*H*W][3C] in qkv's layout; dtable [169][heads] += the bias gradient
// (optional); scratch holds grid_attention_bwd_scratch_floats(N, H, heads) fp32
cudaError_t launch_grid_attention_bwd(const __nv_bfloat16* qkv, const float* table, const __nv_bfloat16* o,
                                      const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv, float* dtable,
                                      float* scratch, int N, int H, int W, int heads, int C, bool grid, float scale,
                                      cudaStream_t stream);
size_t grid_attention_bwd_scratch_floats(int N, int H, int heads);

// ---- Swin V2: scaled-cosine shifted-window attention, window 8, head dim 32 (window_attention_v2.cu) -------------------
// qkv [N*H*W][3C] bf16 in image order (head h: Q, K, V at columns 32h, C + 32h, 2C + 32h), C = 32 heads, any H, W (the
// windows tile the padded frame ceil(H/8) 8 x ceil(W/8) 8; a padding token has q = qb, k = 0, v = vb: fp32 [C] or null),
// shift (sy, sx) in [0, 8) (0 on a side whose padded size is 8).  forward: o [N*H*W][C] and lse [N*H*W][heads] fp32 with
// logits cos(q, k) exp(min(scale[h], ln 100)) + table[225][heads] + the shifted-window mask.
cudaError_t launch_window_attention_v2_fwd(const __nv_bfloat16* qkv, const float* table, const float* scale,
                                           const float* qb, const float* vb, __nv_bfloat16* o, float* lse, int N, int H,
                                           int W, int heads, int C, int sy, int sx, cudaStream_t stream);
// backward (three kernels, deterministic): dqkv [N*H*W][3C] in qkv's layout; dtable [225][heads] = the table gradient,
// dscale [heads] += the logit-scale gradient, dbias [3C] q / v slices += the bias gradients (over every token, padding
// included, or with bias_pad_only over the padding tokens only; the k slice is not touched), each optional; scratch
// holds window_attention_v2_bwd_scratch_floats(N, H, heads) fp32
cudaError_t launch_window_attention_v2_bwd(const __nv_bfloat16* qkv, const float* table, const float* scale,
                                           const float* qb, const float* vb, const __nv_bfloat16* o,
                                           const __nv_bfloat16* dout, const float* lse, __nv_bfloat16* dqkv,
                                           float* dtable, float* dscale, float* dbias, float* scratch, int N, int H,
                                           int W, int heads, int C, int sy, int sx, bool bias_pad_only,
                                           cudaStream_t stream);
size_t window_attention_v2_bwd_scratch_floats(int N, int H, int heads);

// ---- Swin V2: continuous position bias and the patch-merging gather (swin_v2.cu) --------------------------------------
// table [225][heads] = 16 sigmoid(W2 relu(W1 coords[k] + b1)) (coords [225][2], W1 [512][2], b1 [512], W2 [heads][512],
// heads <= 32); with qkv_b_eff, also qkv_b_eff [3C] = qkv_b with its k slice zeroed.  One launch.
cudaError_t launch_cpb_fwd(const float* coords, const float* w1, const float* b1, const float* w2, float* table,
                           const float* qkv_b, float* qkv_b_eff, int heads, int C, cudaStream_t stream);
// dw1 [512][2], db1 [512], dw2 [heads][512] += the gradients from dtable [225][heads] and the forward's table (each
// optional; two launches, fixed order); scratch holds cpb_bwd_scratch_floats(heads) fp32
cudaError_t launch_cpb_bwd(const float* coords, const float* w1, const float* b1, const float* w2, const float* table,
                           const float* dtable, float* dw1, float* db1, float* dw2, float* scratch, int heads,
                           cudaStream_t stream);
size_t cpb_bwd_scratch_floats(int heads);
// forward: dst [N * H/2 * W/2][4C] = the 2x2 gather (x0, x1, x2, x3) of src [N][H][W][C]; backward: src [rows][4C] -> dst
// [N][H][W][C] (H, W even, C % 8 == 0)
cudaError_t launch_merge_gather(const __nv_bfloat16* src, __nv_bfloat16* dst, int N, int H, int W, int C, bool forward,
                                int sms, cudaStream_t stream);

// ---- Swin: patch merging (swin.cu) -------------------------------------------------------------------------------------
// y [N * H/2 * W/2][4C] = LayerNorm over 4C of the 2x2 gather (x0, x1, x2, x3) of the NHWC x [N][H][W][C] (H, W even,
// C % 8 == 0, C <= 512), saving fp32 mean / rstd [rows]
cudaError_t launch_patch_merge_fwd(const __nv_bfloat16* x, const float* gamma, const float* beta, __nv_bfloat16* y,
                                   float* mean, float* rstd, int N, int H, int W, int C, float eps, int sms,
                                   cudaStream_t stream);
// dx [N][H][W][C] of the forward from dy [rows][4C]; dgamma / dbeta [4C] += fixed-order sums (optional, two kernels);
// scratch holds patch_merge_bwd_blocks(sms) * 8C fp32
cudaError_t launch_patch_merge_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, const float* mean, const float* rstd,
                                   const float* gamma, __nv_bfloat16* dx, float* dgamma, float* dbeta, float* scratch,
                                   int N, int H, int W, int C, int sms, cudaStream_t stream);
int patch_merge_bwd_blocks(int sms);

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
// hardswish on n bf16 elements (n % 8 == 0) and its backward from the saved pre-activation x
cudaError_t launch_hardswish_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, cudaStream_t stream);
cudaError_t launch_hardswish_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* x, __nv_bfloat16* dx, int64_t n,
                                 cudaStream_t stream);
// ---- squeeze-excitation (squeeze_excite.cu) -------------------------------------------------------------------
// x / y / dy / dx [N][HW][C] bf16 (C % 8 == 0); s = fc2 output [N][lds] bf16 (pre-hardsigmoid, lds % 8 == 0)
// y = x * hsig(s)
cudaError_t launch_se_scale(const __nv_bfloat16* x, const __nv_bfloat16* s, int lds, __nv_bfloat16* y, int N, int HW,
                            int C, int sms, cudaStream_t stream);
// ds [N][ldd] = hsig'(s) * sum_hw(dy * x), columns [C, ldd) zero (ldd <= C rounded up to 64); deterministic
cudaError_t launch_se_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* s, int lds,
                             __nv_bfloat16* ds, int ldd, int N, int HW, int C, cudaStream_t stream);
// dx = dy * hsig(s) + dpooled / HW  (dpooled [N][C])
cudaError_t launch_se_apply(const __nv_bfloat16* dy, const __nv_bfloat16* s, int lds, const __nv_bfloat16* dpooled,
                            __nv_bfloat16* dx, int N, int HW, int C, int sms, cudaStream_t stream);
// ---- squeeze-excitation with a sigmoid gate (squeeze_excite_sigmoid.cu; EfficientNet) -------------------------------
// same operands as above; gate sigmoid(s), reduce ds = g (1 - g) * sum_hw(dy * x)
cudaError_t launch_se_sig_scale(const __nv_bfloat16* x, const __nv_bfloat16* s, int lds, __nv_bfloat16* y, int N, int HW,
                                int C, int sms, cudaStream_t stream);
cudaError_t launch_se_sig_reduce(const __nv_bfloat16* dy, const __nv_bfloat16* x, const __nv_bfloat16* s, int lds,
                                 __nv_bfloat16* ds, int ldd, int N, int HW, int C, cudaStream_t stream);
cudaError_t launch_se_sig_apply(const __nv_bfloat16* dy, const __nv_bfloat16* s, int lds, const __nv_bfloat16* dpooled,
                                __nv_bfloat16* dx, int N, int HW, int C, int sms, cudaStream_t stream);
// Batched zero padding: each matrix src [rows][k] (bf16 or fp32: esize 2 / 4) -> dst [prows][kp] with src in the
// top-left corner and zeros elsewhere (fc2's squeeze dimension padded to 8; ShuffleNetV2's operands padded to 8 in both
// dimensions), one launch for up to kPadMax matrices
constexpr int kPadMax = 24;
struct PadMatrix {
  const void* src;
  void* dst;
  int rows, k, prows, kp, esize;
};
struct PadBatch {
  PadMatrix m[kPadMax];
  int n;
};
cudaError_t launch_pad_cols(const PadBatch& b, cudaStream_t stream);
// Batched fold: fp32 dst [rows][k] += src [>= rows][kp] columns [0, k) (add), or = (copy: running statistics)
struct FoldMatrix {
  const void* src;
  void* dst;
  int rows, k, kp, add;
};
struct FoldBatch {
  FoldMatrix m[kPadMax];
  int n;
};
cudaError_t launch_fold_cols(const FoldBatch& b, cudaStream_t stream);
// SiLU on the rows of a bf16 matrix: y [N][ldy] = silu(x [N][ldx]) for columns [0, ldy) (ldy <= ldx, both % 8 == 0), and
// its backward dx [N][ldx] = dy [N][ldy] * silu'(x) for columns < c_valid, zero elsewhere (a GEMM operand with zero pad)
// tanh on n bf16 elements (n % 8 == 0), and dx = dy * (1 - y^2) from the saved output y
cudaError_t launch_tanh_rows_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int64_t n, cudaStream_t stream);
cudaError_t launch_tanh_rows_bwd(const __nv_bfloat16* dy, const __nv_bfloat16* y, __nv_bfloat16* dx, int64_t n,
                                 cudaStream_t stream);
cudaError_t launch_silu_rows_fwd(const __nv_bfloat16* x, int ldx, __nv_bfloat16* y, int ldy, int N, cudaStream_t stream);
cudaError_t launch_silu_rows_bwd(const __nv_bfloat16* dy, int ldy, const __nv_bfloat16* x, int ldx, __nv_bfloat16* dx,
                                 int c_valid, int N, cudaStream_t stream);
// stochastic depth: keep[i] = (uniform(seed, step, offset + i) > p) / (1 - p) for i < n, from the dropout Philox stream
cudaError_t launch_stochastic_depth_keep(float* keep, int n, float p, uint64_t seed, uint64_t offset, const int64_t* step,
                                         cudaStream_t stream);
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

// ---- ShuffleNetV2: channel shuffle fused into the branch BatchNorm (shufflenet.cu) ----------------------------------
// s[2i] = a[i] (stride 1: the pass-through, a bit copy) or relu(BN_a(a[i])) (stride 2), s[2i+1] = relu(BN_b(b[i])),
// i < half (even).  a, b and the backward outputs da, db: [M][ld_ab]; s whole [M][ld_s] or its halves lo = s[:, :half],
// hi = s[:, half:] ([M][ld_ab] each, split).  Channels past the real width are written as zeros.
struct ShuffleBn {
  const float* sum;          // train forward: per-channel sum / sum of squares of the conv output (conv epilogue)
  const float* sumsq;
  const float* gamma;        // [half]
  const float* beta;
  float* mean;               // [half]: written by a train forward, read by backward
  float* invstd;
  float* running_mean;       // [half]: updated by a train forward (may be null), read in eval
  float* running_var;
  float eps, momentum;
  float* dgamma;             // backward: [half] zeroed scratch receiving the sums
  float* dbeta;
  float* gamma_grad;         // backward, optional: accumulate targets
  float* beta_grad;
};
struct ShuffleArgs {
  const __nv_bfloat16* a;    // forward input / backward saved conv output (a_bn only)
  const __nv_bfloat16* b;
  __nv_bfloat16* s0;         // forward output: s, or lo
  __nv_bfloat16* s1;         //   hi (split)
  const __nv_bfloat16* ds0;  // backward input: ds, or dlo
  const __nv_bfloat16* ds1;  //   dhi (split)
  __nv_bfloat16* da;         // backward output: the pass-through gradient (stride 1) or BN_a's input gradient
  __nv_bfloat16* db;         //   BN_b's input gradient
  int M, half, ld_ab, ld_s;  // ld_s: row pitch of s, or of lo / hi (= ld_ab)
  int split, a_bn, train;
  ShuffleBn bn_a, bn_b;
};
cudaError_t launch_shuffle_fwd(const ShuffleArgs& p, int sms, cudaStream_t stream);
// two launches: the reduce pass (and the pass-through copy), then the apply pass
cudaError_t launch_shuffle_bwd(const ShuffleArgs& p, int sms, cudaStream_t stream);

// ---- GoogLeNet: segmented BatchNorm + ReLU, adaptive average pooling, row transpose (inception.cu) ---------------
// One launch applies up to kSegMax BatchNorm + ReLU layers, each to a channel segment of C (% 8 == 0) channels read
// from x[r * ldx + colx + c] and written to z[r * ldz + colz + c] (forward), or with the gradient read from
// dz[r * lddz + coldz + c] and written to dx[r * lddx + coldx + c] (backward, x the saved pre-BN input).  Pitches and
// column offsets are multiples of 8; channels of a destination outside its segment are not touched.
constexpr int kSegMax = 4;
struct BnSeg {
  const __nv_bfloat16* x;
  __nv_bfloat16* z;
  const __nv_bfloat16* dz;
  __nv_bfloat16* dx;
  int ldx, colx, ldz, colz, lddz, coldz, lddx, coldx;
  int C;
  const float* sum;          // train forward: the conv epilogue's per-channel sum / sum of squares
  const float* sumsq;
  const float* gamma;
  const float* beta;
  float* mean;               // written by a train forward, read by backward
  float* invstd;
  float* running_mean;       // updated by a train forward (may be null), read in eval
  float* running_var;
  float eps, momentum;
  float* dgamma;             // backward: this step's dgamma / dbeta (written by the reduce pass, read by the apply pass)
  float* dbeta;
  float* gamma_grad;         // backward, optional: accumulate targets (the .grad slots)
  float* beta_grad;
};
struct BnSegArgs {
  BnSeg s[kSegMax];
  int n, M;
  int chunk0[kSegMax + 1];   // first 64-channel chunk of each segment (set by the launchers)
  float* partial;            // backward: [chunks][grid_x][128] per-block sums
  unsigned int* done;        // backward: [chunks] zeroed counters (left zeroed)
};
// blocks along the rows of the segmented kernels for `chunks` 64-channel chunks (the backward's partial buffer holds
// chunks * bn_seg_grid_x(...) * 128 floats)
int bn_seg_grid_x(int M, int chunks, int sms);
cudaError_t launch_bn_seg_fwd(BnSegArgs a, bool train, int sms, cudaStream_t stream);
// two launches: the reduce pass (dgamma / dbeta, deterministic), then the apply pass
cudaError_t launch_bn_seg_bwd(BnSegArgs a, int grid_x, cudaStream_t stream);
// NHWC [N][H][W][C] <-> [N][P][Q][C] with torch's adaptive windows; C % 8 == 0
cudaError_t launch_adaptive_avgpool_fwd(const __nv_bfloat16* x, __nv_bfloat16* y, int N, int H, int W, int C, int P,
                                        int Q, int sms, cudaStream_t stream);
cudaError_t launch_adaptive_avgpool_bwd(const __nv_bfloat16* dy, __nv_bfloat16* dx, int N, int H, int W, int C, int P,
                                        int Q, int sms, cudaStream_t stream);
// out[n][b][a] = in[n][a][b], A % 8 == 0
cudaError_t launch_transpose_rows(const __nv_bfloat16* in, __nv_bfloat16* out, int N, int A, int B, int sms,
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
