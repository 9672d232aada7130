// Which kernel runs a convolution, and how it is launched.  conv_plan (conv_tc.cu) makes the choice for one call from
// the descriptor and the facts listed in ConvCall, in host arithmetic only; the entry points of api.cu launch the family
// it names, and se_conv2d_path / se_conv2d_plan report it, so that the query and the launch cannot differ.
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
  int box_tiles;               // > 0: 3x3 / stride 1 with X staged once per CTA, this many 64-row tiles per CTA
  float* ws;                   // [2 * gridDim.x][KK * Cout] partial dW, then [2 * gridDim.x][Cout] partial dbias
  float* dw;                   // direct mode (ws == nullptr): atomics straight into dW / dbias
  float* dbias;
};

// conv_odd_tc_kernel: forward (flip 0) or data gradient (flip 1) of a 3x3 / stride 1 / 'same' layer, any channel counts
struct OddTcParams {
  int H, W, npx;            // image rows and pixels, N * H * W
  int Kc, Nc;               // GEMM K channels (A tensor channels), GEMM N channels (output channels)
  int flip;                 // 1: dgrad (B = the HWIO kernel, tap order reversed)
  int relu;
  float beta;               // out = beta * out + D (dgrad; 0 in the forward pass)
  const float* bias;
  const float* residual;
  float* out;
};

// conv_odd_wgrad_tc_kernel: split z sums the pixels [z * per_split, (z + 1) * per_split)
struct OddWgParams {
  int H, W, Cin, Cout, npx, per_split;
  float* ws;                   // [gridDim.z][9 * Cin * Cout] partial dW, then [gridDim.z][Cout] partial dbias
  float* dw;                   // direct mode (ws == nullptr): atomics straight into dW / dbias
  float* dbias;
};

// conv_simt.cu
struct SimtParams {
  int bn;                   // conv_fwd_kernel / conv_dgrad_kernel tile by its BN: <128, 16, 4, 2>, <128, 32, 4, 4>, <64, 64, 4, 4>
  int vec;                  // ... with float4 loads
  int par;                  // conv_dgrad_kernel: rows ordered by stride-2 parity class
  int nci, nco;             // conv_wgrad3x3_kernel<NCI, NCO>
  int TH, PG;               // image rows per tile (stems, conv_wgrad3x3_kernel); pixel groups (conv_wgrad_stem_kernel)
  int tiles_per_img, num_tiles;
  long long per;            // conv_wgrad_kernel: pixels per split
};

enum ConvFamily {
  CONV_FP32_TILES,       // conv_simt.cu: conv_fwd_kernel / conv_dgrad_kernel
  CONV_FP32_DENSE_SMALL, // dense_small_fwd_kernel
  CONV_FP32_FWD_STEM,    // conv_fwd_stem_kernel
  CONV_FP32_WGRAD,       // conv_wgrad_kernel
  CONV_FP32_WGRAD_STEM,  // conv_wgrad_stem_kernel
  CONV_FP32_WGRAD_3X3,   // conv_wgrad3x3_kernel<NCI, NCO>
  CONV_TC_3X3,           // conv_tc_kernel: 3x3 / stride 1 / 'same'
  CONV_TC_1X1,           // conv_tc_kernel: 1x1 / stride 1, the flat pixel list
  CONV_TC_1X1_S2,        // conv_tc_kernel: 1x1 / stride 2 through the sub-sampled view
  CONV_TC_DGRAD_3X3S2,   // data gradient of a wide 3x3 / stride 2 layer: nine 1x1 / stride 2 launches, one per tap
  CONV_TC_WGRAD,         // conv_wgrad_tc_kernel
  CONV_TC_ODD_3X3,       // conv_odd_tc.cu: 3x3 / stride 1 / 'same' with channel counts that are not multiples of 8
};
inline bool conv_is_tc(ConvFamily f) { return f >= CONV_TC_3X3; }

// The facts about one call that the choice depends on, besides descriptor, direction and mode.  The defaults are what
// se_conv2d_path assumes.
struct ConvCall {
  bool w_t = true, w_t_lo = true, w_lo = true;   // the auxiliary kernel copies of se_conv_aux that are present
  bool stats = false;                             // forward: BatchNorm statistics requested
  float beta = 0.f;                               // backward data: dx = beta * dx + dX
  bool aligned = true;                            // weight gradient: dw and dbias 16-byte aligned
  bool x_aligned = true;                          // forward: x 16-byte aligned (dense_small_fwd_kernel)
  bool y_aligned = true;                          // forward: y 16-byte aligned (conv_fwd_stem_kernel)
  bool dy_aligned = true;                         // weight gradient: dy 16-byte aligned (conv_wgrad_stem_kernel)
  bool residual = false;                          // forward: a residual is added
  int sms = 0;                                    // SMs of the device (0: unknown): grids, split-K slices
};

struct ConvPlan {
  ConvFamily family = CONV_FP32_TILES;
  int x3 = 0;                 // error-compensated arithmetic (3xTF32)
  bool fused_stats = false;   // forward with statistics: summed in the epilogue, else by a separate se_bn_stats pass
  dim3 grid, block;           // block: the fp32 kernels (the tensor-core kernels have a fixed thread count)
  size_t smem = 0;
  // weight gradient: split-K slices of the workspace (wgrad_workspace), added into dW / dbias in slice order; they
  // fix the order of the sums, so every family's rule for them must stay as it is (DESIGN §5.1)
  long long splits = 0;
  long long split_px = 0;     // pixels of each CTA's range of the split (0: CTAs stride over image tiles)
  SimtParams fp = {};         // conv_simt.cu
  ConvTcParams tc = {};       // conv_tc_kernel: every field but relu and the pointers
  WgTcParams wg = {};         // conv_wgrad_tc_kernel: every field but the pointers
  int wg_bn = 0, wg_np = 1;   // conv_wgrad_tc_kernel<BN, X3, NP>
  OddTcParams od = {};        // conv_odd_tc_kernel: every field but relu, beta and the pointers
  OddWgParams owg = {};       // conv_odd_wgrad_tc_kernel: every field but the pointers
  int od_bn = 0;              // N tile of the conv_odd_tc kernels (32 or 64)
};

// dir 0 forward, 1 backward data, 2 weight gradient; the descriptor is valid (check_desc)
ConvFamily conv_plan(const se_conv_desc* d, int dir, int mode, const ConvCall& call, ConvPlan* p);
void simt_config(const se_conv_desc* d, int dir, const ConvCall& call, ConvPlan* p);   // the fp32 families

// Where a weight-gradient kernel puts its split-K partial sums: the slices of the workspace, or dW / dbias themselves
// with float atomics (direct mode: ws == nullptr)
struct WgOut {
  float* ws;                  // the workspace, or nullptr
  float* dw;                  // ws, or dW
  float* dbias;               // the bias slices (after every dW slice), or dbias; nullptr: no bias gradient
};

int conv_fwd_simt(const ConvPlan& p, const se_conv_desc* d, const float* x, const float* w, const float* bias,
                  const float* residual, float* y, int relu, double* stats, cudaStream_t st);
int conv_dgrad_simt(const ConvPlan& p, const se_conv_desc* d, const float* dy, const float* w, float* dx, float beta,
                    cudaStream_t st);
int conv_wgrad_simt(const ConvPlan& p, const se_conv_desc* d, const float* x, const float* dy, const WgOut& o,
                    cudaStream_t st);

int conv_fwd_tc(const ConvPlan& p, const se_conv_desc* d, const float* x, const float* w_t, const float* w_t_lo,
                const float* bias, const float* residual, float* y, int relu, double* stats, cudaStream_t st);
int conv_dgrad_tc(const ConvPlan& p, const se_conv_desc* d, const float* dy, const float* w, const float* w_lo, float* dx,
                  float beta, cudaStream_t st);
int conv_wgrad_tc(const ConvPlan& p, const float* x, const float* dy, const WgOut& o, cudaStream_t st);
int conv_fwd_odd_tc(const ConvPlan& p, const float* x, const float* w_t, const float* w_t_lo, const float* bias,
                    const float* residual, float* y, int relu, cudaStream_t st);
int conv_dgrad_odd_tc(const ConvPlan& p, const float* dy, const float* w, const float* w_lo, float* dx, float beta,
                      cudaStream_t st);
int conv_wgrad_odd_tc(const ConvPlan& p, const float* x, const float* dy, const WgOut& o, cudaStream_t st);

}  // namespace se
