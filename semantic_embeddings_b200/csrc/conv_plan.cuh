// Which kernel runs a convolution, and how it is launched.  conv_plan (conv_tc.cu) makes the choice for one call from
// the descriptor and the facts listed in ConvCall, in host arithmetic only; the entry points of api.cu launch the family
// it names, and se_conv2d_path reports it, so that the query and the launch cannot differ.
#pragma once
#include "common.cuh"

namespace se {

struct ConvTcParams {
  int N, H, W;              // extent of the grid the pixel tiles cover (images, rows, pixels)
  int Kc, Nc, BN;           // GEMM K channels (A tensor channels), GEMM N channels, output channels per tile
  int Wb, Hb, Nb;           // pixel box, Wb*Hb*Nb == 128
  int tw, th;               // tiles along a row / along the rows of an image
  int cblk, kblocks;        // channels per pipeline stage (16 or 32), Kc / cblk
  int taps, pad, flip;      // filter size (3 or 1), 'same' padding rows (1 or 0), 1: dgrad (tap order reversed for B)
  int res;                  // 1: resident box (A loaded once per tile, stages hold B only), 0: per-tap stages
  int ring_off;             // bytes of shared memory before the stage ring (the resident box)
  int stages, stage_bytes, b_bytes;   // stage = [A of one tap (per-tap only)] B [B_lo (X3)]
  int a_bytes, a_tx;        // one A tile (per-tap stage / channel block of the resident box): slot size, TMA bytes
  long long o_sn, o_sh, o_sw;   // output (and residual) element strides of an image, a row, a pixel
  int ovh, ovw;             // rows / pixels of the output view that exist (a strided view may be one short)
  int relu;
  float beta;               // dgrad: out = beta*out + D
  const float* bias;
  const float* residual;
  float* out;
  double* stats;
};

struct WgTcParams {
  int N, H, W, Cin, Cout, Ho, Wo, kw, stride, pad_t, pad_l;
  int KK;                      // rows of dW: kh * kw * Cin, row = tap * Cin + ci
  int npx;                     // N * Ho * Wo
  int chunks;                  // ceil(npx / 32)
  int per_cta;                 // chunks per CTA (even)
  float* ws;                   // [2 * gridDim.x][KK * Cout] partial dW, then [2 * gridDim.x][Cout] partial dbias
  float* dw;                   // direct mode (ws == nullptr): atomics straight into dW / dbias
  float* dbias;
};

enum ConvFamily {
  CONV_FP32,             // conv_simt.cu
  CONV_TC_3X3,           // conv_tc_kernel: 3x3 / stride 1 / 'same'
  CONV_TC_1X1,           // conv_tc_kernel: 1x1 / stride 1, the flat pixel list
  CONV_TC_1X1_S2,        // conv_tc_kernel: 1x1 / stride 2 through the sub-sampled view
  CONV_TC_DGRAD_3X3S2,   // data gradient of a wide 3x3 / stride 2 layer: nine 1x1 / stride 2 launches, one per tap
  CONV_TC_WGRAD,         // conv_wgrad_tc_kernel
};

// The facts about one call that the choice depends on, besides descriptor, direction and mode.  The defaults are what
// se_conv2d_path assumes.
struct ConvCall {
  bool w_t = true, w_t_lo = true, w_lo = true;   // the auxiliary kernel copies of se_conv_aux that are present
  bool stats = false;                             // forward: BatchNorm statistics requested
  float beta = 0.f;                               // backward data: dx = beta * dx + dX
  bool aligned = true;                            // weight gradient: dw and dbias 16-byte aligned
  int sms = 0;                                    // weight gradient: SMs of the device; sizes the split-K grid only
};

struct ConvPlan {
  ConvFamily family = CONV_FP32;
  int x3 = 0;                 // error-compensated arithmetic (3xTF32)
  bool fused_stats = false;   // forward with statistics: summed in the epilogue, else by a separate se_bn_stats pass
  dim3 grid;
  size_t smem = 0;
  ConvTcParams tc = {};       // conv_tc_kernel: every field but relu and the pointers
  WgTcParams wg = {};         // conv_wgrad_tc_kernel: every field but the pointers
  int wg_bn = 0, wg_np = 1;   // conv_wgrad_tc_kernel<BN, X3, NP>
};

// dir 0 forward, 1 backward data, 2 weight gradient; the descriptor is valid (check_desc)
ConvFamily conv_plan(const se_conv_desc* d, int dir, int mode, const ConvCall& call, ConvPlan* p);

int conv_fwd_tc(const ConvPlan& p, const se_conv_desc* d, const float* x, const float* w_t, const float* w_t_lo,
                const float* bias, const float* residual, float* y, int relu, double* stats, cudaStream_t st);
int conv_dgrad_tc(const ConvPlan& p, const se_conv_desc* d, const float* dy, const float* w, const float* w_lo, float* dx,
                  float beta, cudaStream_t st);
int conv_wgrad_tc(const ConvPlan& p, const float* x, const float* dy, float* dw, float* dbias, cudaStream_t st);

}  // namespace se
