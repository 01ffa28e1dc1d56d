// Host/device shared argument structs for the wgmma implicit-GEMM convolution kernels.
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ddl {

enum ConvMode : int {
  kConvFwd = 0,        // A = im2col(x) gathered with cp.async, rows = output pixels (any stride / dilation)
  kConvDgrad = 1,      // A = transposed-conv gather of dy, rows = input pixels, B is MN-major (any stride)
  kConvGemm = 2,       // A is a plain [M][K] matrix fetched by 2-D TMA (1x1 stride-1 convs, FC)
  kConvStem = 3,       // small-Cin first conv on a 4-channel image: k-block = RPK filter rows x SP taps x 4 ch
  kConvTileFwd = 4,    // stride-1 conv: A tile = rectangle of output pixels fetched by ONE 4-D TMA box per tap
                       //   (padding = TMA out-of-bounds zero fill), rows = (n, h, w) of the rectangle
  kConvTileDgrad = 5,  // same for the data gradient of a stride-1 conv (source = dy, B MN-major)
  kConvGemmDgrad = 6,  // 1x1 stride-1 data gradient: A = dy matrix via 2-D TMA, B MN-major
  kConvStemTma = 7,    // small-Cin first conv with an EVEN stride on a zero-padded NHWC4 image: the k-block of a
                       //   row (RPK filter rows x SP taps x 4 ch = 128 B) is ONE box of a 5-D tensor map whose
                       //   dimensions overlap in memory: (tap*ch | filter row | out col | out row | image) with
                       //   strides (1 | Wp*4 | stride*4 | stride*Wp*4 | Hp*Wp*4) elements.  Replaces 64 8-byte
                       //   cp.async per output pixel of kConvStem by 4 TMA requests per 128-pixel tile.
};

struct ConvArgs {
  const __nv_bfloat16* src;   // gather source (x for fwd / stem, dy for dgrad); unused for TMA-A modes
  __nv_bfloat16* out;         // [M][ldc] (NHWC activations / gradients)
  const __nv_bfloat16* add;   // optional: out = acc + add   (same layout as out)
  const uint8_t* add_mask;    // optional with `add`: bit i of byte [m][c/8] gates add[m][c + i] (the ReLU bit mask
                              //   of the block output: the shortcut gradient dz * (z > 0) is formed here instead
                              //   of being written by the BN-backward kernel and read back)
  const float* bias;          // optional: per output channel
  float* sum;                 // optional BN statistics: sum[c]   += sum_m out[m][c]   (of the bf16-rounded value)
  float* sumsq;               //                         sumsq[c] += sum_m out[m][c]^2
  // optional (dgrad launches): fuse the BatchNorm-backward reduction of the layer whose output gradient this kernel
  // produces.  With bnr_y != nullptr the statistics epilogue accumulates, per channel of `out`,
  //   sum[c] += S1 = sum_m dm,   sumsq[c] += invstd[c] * (S2 - mean[c] * S1),  S2 = sum_m dm * y[m][c]
  // where dm = out[m][c] * [gamma*invstd*(y - mean) + beta > 0] — i.e. dbeta and dgamma of that BN (ReLU mask
  // recomputed from its saved input y), so the separate reduce pass over (d, y) is not needed.
  // With `bnr_mask` the ReLU mask comes from that BN's forward bit mask instead (a residual layer: its output includes
  // the shortcut); with `add` (linear rows only) the sums are taken over the stored value acc + gated add.
  const __nv_bfloat16* bnr_y;
  const uint8_t* bnr_mask;
  const float* bnr_gamma;
  const float* bnr_beta;
  const float* bnr_mean;
  const float* bnr_invstd;
  int M;                      // GEMM rows (= batch * dstH * dstW)
  int KB;                     // number of 64-element k-blocks
  int ldc;                    // channels of `out` (row stride in elements)
  int srcH, srcW, srcC;       // gather-source geometry
  int dstH, dstW;             // GEMM-row geometry
  int R, S, stride, pad, dil; // pad = padding along H
  int pad_w;                  // padding along W (asymmetric 1x7 / 7x1 kernels)
  int cchunks;                // ceil(srcC / 64) k-blocks per filter tap (stem: padded taps per filter row)
  int kstride;                // K-major weights: elements between consecutive taps in a weight row (= true Cin).
                              //   srcC need not be a multiple of 64: the last k-block of a tap is zero-filled on
                              //   the activation side (TMA out-of-bounds / masked gather), so whatever weight
                              //   columns the B box picks up beyond the tap contribute nothing.
  int relu;                   // apply ReLU in the epilogue (after bias)
  int n_valid;                // output channels that really exist (bias is read only below this)
  int stages;                 // pipeline depth actually used (<= compile-time maximum)
  // FP8 operands (deep-ring kernel only): 0 = bf16; 1 = A and B are e4m3; 2 = A is e5m2 (gradients), B is e4m3.
  // A k-block is still 128 BYTES per row (128 fp8 elements), so shared-memory images, swizzle and descriptors keep
  // their geometry; tensor maps are built over bytes.  The epilogue multiplies the accumulator by *deq_a * *deq_b
  // (the operands' inverse quantisation scales, device-resident: ops.h Fp8Slot::inv_scale).
  int fp8;
  const float* deq_a;
  const float* deq_b;
  // MX block scales (unused by the sm_90a kernels, which have no block-scaled MMA; the launcher rejects fp8 = 3)
  const uint8_t* sfa;
  const uint8_t* sfb;
  int variant;                // kernel variant word chosen by the caller's autotuner (0 = built-in policy); see
                              //   launch_fwd_mode in conv_gemm.cu for the encoding
  // tile modes: the M tile is a tw x th x tn box of pixels of the dstH x dstW iteration grid (w fastest);
  // tw*th*tn <= 128.  Row (n, i, j) of the grid is written to out[n][out_stride*i + out_pa][out_stride*j + out_pb]
  // of an outH x outW image (dense output: out_stride = 1).
  int batch, tw, th, tn, tiles_w, tiles_h;
  int outH, outW, out_stride, out_pa, out_pb;
  int zfill;                  // stride-2 scatter with a single live phase: also write zeros to the 3 sibling pixels
  // optional explicit tap table (strided convs decomposed into stride-1 phase problems): per tap the box offset
  // in the source map, which of the 4 source maps to read, and the weight tap index r*S+s
  int ntaps;
  signed char tap_dh[16], tap_dw[16], tap_map[16], tap_widx[16];
  // grouped convolution (Cin = Cout = C): 0 = dense, else the bundle width Wb.  A bundle is max(1, 64 / cg)
  // consecutive groups (Wb channels) and spans T = ceil(Wb / 64) = cchunks N tiles of 64 and T k-blocks per filter tap
  // (KB = R*S*T).  N tile nt (expanded row n0 = 64 nt) is slice t = nt % T of bundle b = nt / T: it writes channels
  // [b*Wb + 64 t, min(b*Wb + 64 t + 64, (b + 1)*Wb, C)) and reads source channels b*Wb + [0, 64 T).  The weights are
  // the expanded matrix [nbundles*T*64][R*S*T*64] (expand_grouped_weight), zero outside each bundle's groups: K-major
  // with kstride = 64 T in the forward, MN-major rows (b*T + cc)*64 x columns (tap*T + t)*64 in the data gradient.
  int grouped;
};

struct TmaSet {          // up to 4 activation maps (the 2x2 phase sub-images of a stride-2 source)
  CUtensorMap m[4];
};

struct WgradArgs {
  const __nv_bfloat16* x;     // gather source for the B operand (im2col(x)), NHWC
  float* dw;                  // fp32 accumulator [Cout][ldw]  (split-K: red.add)
  int M;                      // pixels = batch * P * Q  (GEMM reduction dim)
  int Cout;
  int dy_ld;                  // row stride (elements) of dy; >= Cout (padded FC logits)
  int ldw;                    // row stride of dw = R*S*Cin (or 256 for the stem scratch)
  int ncols;                  // columns of the virtual (tap, Cpad) space = R*S*Cpad (stem / GEMM: real columns)
  int H, W, C;                // x geometry
  int P, Q;                   // dy geometry
  int R, S, stride, pad, dil;
  int pad_w;
  int cchunks;                // stem only: padded taps per filter row
  int Cpad;                   // virtual channels per tap = C rounded up to 64: tile columns are indexed (tap, c) in
  int Cw;                     //   this padded space; Cw = real channels per tap of the dw row (dw col = tap*Cw + c)
  int kb_per_split;           // pixel blocks handled by one CTA
  int total_kb;               // number of pixel blocks
  int mode;                   // kConvFwd (gather), kConvGemm (x via 2-D TMA), kConvStem, kConvTileFwd (4-D TMA)
  int stages;
  int batch, tw, th, tn, tiles_w, tiles_h;   // tile mode: a pixel block is a tw x th x tn box (<= 64 pixels)
  int group_width;            // grouped convolution: input channels per group (0 = dense).  Tiles are 64 output
                              //   channels (slice t of a bundle, see ConvArgs::grouped) x (tap, the bundle's 64 T input
                              //   channels) (Cpad = 64 T); only the in-group entries are added, to dw column
                              //   tap * group_width + ci % group_width
};

}  // namespace ddl
