/* se_b200.h -- C ABI of the H100-native hot path of cvjena/semantic-embeddings.
 *
 * The reference (/root/reference, pure Python on Keras 2.2 / TF 1.x) has no FFI layer: its
 * device work is whatever the Keras graph of learn_image_embeddings.py and the numpy calls of
 * evaluate_retrieval.py:56-67 dispatch to cuDNN/cuBLAS/BLAS.  Each entry point below replaces
 * one group of those graph ops; the comment on each names the reference lines it stands for.
 * The host side (the semantic_embeddings_b200 package) binds this file with ctypes; INTEGRATION.md shows
 * the binding a maintainer of the reference would add.
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no torch / C++ types.
 *   - every function returns 0 on success, <0 on error (SE_ERR_*); se_last_error() gives the
 *     message of the calling thread's last failure.
 *   - device pointers are caller-owned (PyTorch tensors are used as containers); the library
 *     never allocates or frees device memory.  Kernels that need scratch take it explicitly.
 *   - `stream` is a cudaStream_t; all calls are asynchronous w.r.t. the host and capturable
 *     into a CUDA graph.
 *   - process-wide state is limited to what se_init() / se_comm_init() create: the low-priority
 *     side stream and the fork/join events se_run_ops uses for weight gradients, and the NCCL
 *     communicator with its stream.  Kernels keep no state between calls.
 *   - activations are float32 NHWC; conv kernels are float32 HWIO (Keras layout); dense
 *     kernels are (in,out).  `mode` selects the arithmetic of contraction kernels:
 *     SE_MODE_F32 = fp32 FFMA; SE_MODE_TF32 = TF32 wgmma (operands read with a
 *     10-bit mantissa, fp32 accumulate: ~1e-3 relative, outside the reference's fp32
 *     semantics, kept for comparison); SE_MODE_TF32X3 = TF32 wgmma with error
 *     compensation (every operand split into hi + lo, hi*hi + hi*lo + lo*hi in one fp32
 *     accumulator: fp32-level results, the mode the training path runs and is benchmarked in).
 *     Shapes the tensor path does not cover fall back to the fp32 kernels -- never to the CPU.
 */
#ifndef SE_B200_H
#define SE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SE_OK 0
#define SE_ERR_ARG (-1)
#define SE_ERR_CUDA (-2)
#define SE_ERR_UNSUPPORTED (-3)

#define SE_MODE_F32 0
#define SE_MODE_TF32 1
#define SE_MODE_TF32X3 2

/* head variants: learn_image_embeddings.py --loss (lines 62, 127-130, 164-171) */
#define SE_LOSS_INV_CORR 0     /* l2norm wrapper + 1 - <t,x>      */
#define SE_LOSS_UNNORM_CORR 1  /* no wrapper     + 1 - <t,z>      */
#define SE_LOSS_MSE 2          /* no wrapper     + sum (z-t)^2    */
#define SE_LOSS_SOFTMAX_CORR 3 /* softmax wrapper + 1 - <t,x>     (learn_image_embeddings.py:129-130) */
#define SE_LOSS_DEVISE_RANK 4  /* no wrapper     + sum_c relu(m - <t,z> + <z,E_c>) - m   (learn_devise.py; se_devise_rank_fwd_bwd) */

/* pairwise modes: evaluate_retrieval.py:57-62 */
#define SE_PDIST_SQEUCLID 0    /* A + B - 2 F F^T                 */
#define SE_PDIST_NEGDOT 1      /* -(F F^T)  (caller passes normalised F, or sets normalize=1) */

const char* se_version(void);
const char* se_last_error(void);
/* number of kernel launches issued by this library since load (for bench.py's gpu_launches) */
int64_t se_launch_count(void);
int se_device_sm_count(void);
/* one-time per-process setup (device query, shared-memory attributes); call before capturing CUDA graphs */
int se_init(void);
/* bit mask of the tensor-core kernels compiled in: 1 conv fwd, 2 conv dgrad, 4 conv wgrad, 8 pairwise */
int se_tc_capabilities(void);

/* ------------------------------------------------------------------ convolution / dense
 * Conv2D of models/cifar_resnet.py:96-105,218, models/plainnet.py:52,70,
 * models/wide_residual_network.py:9,20,28,31,46,53 and keras.applications.ResNet50 (utils.py:237).
 * Explicit zero padding (pad_t, pad_l) and output size: the host computes TF 'SAME'
 * (pad_before = total//2, so k=3,s=2 on an even input gives pad 0 before / 1 after).
 * In SE_MODE_TF32 / SE_MODE_TF32X3 the tensor-core kernels take: 3x3 / stride 1 / pad 1 on image widths 4..56 (weight
 * gradient: ..64), 1x1 / stride 1 / pad 0 on any image size (>= 128 pixels per call), 1x1 / stride 2 / pad 0 with
 * Wo <= 32 -- channel counts in multiples of 16 (the GEMM K dimension: 16 or a multiple of 32); backward data and weight
 * gradient of 3x3 / stride 2 / pad 0 on even image sizes with >= 128 channels on both sides (nine strided 1x1 GEMMs).
 * Every other shape (3-channel stems, the forward pass and the narrow layers of 3x3 / stride 2, 7x7, dense layers) runs on
 * the fp32 kernels in every mode; se_conv2d_path() tells which. */
typedef struct {
  int32_t N, H, W, Cin;   /* input  NHWC */
  int32_t Cout, kh, kw;   /* kernel HWIO */
  int32_t stride;
  int32_t pad_t, pad_l;
  int32_t Ho, Wo;         /* output NHWC = (N, Ho, Wo, Cout) */
} se_conv_desc;

/* y = conv(x, w) [+ bias] [+ residual] [relu]; optionally accumulates per-channel
 * sum(y) and sum(y^2) (of the stored values) into stats[0:Cout], stats[Cout:2Cout]
 * (float64, caller zeroes) -- the BatchNormalization statistics of the next layer. */
int se_conv2d_fwd(const se_conv_desc* d, const float* x, const float* w, const float* bias,
                  const float* residual, float* y, int relu, double* stats, int mode, void* stream);
/* same, with an optional transposed copy w_t = [kh][kw][Cout][Cin] of the kernel: the tensor-core forward path
 * (SE_MODE_TF32) consumes K-major operands; without w_t the call uses the fp32 kernels. */
int se_conv2d_fwd_ex(const se_conv_desc* d, const float* x, const float* w, const float* w_t, const float* bias,
                     const float* residual, float* y, int relu, double* stats, int mode, void* stream);
/* Auxiliary copies of a convolution kernel w (HWIO) that the tensor-core paths consume; any may be NULL (the call
 * then uses the fp32 kernels):  w_t = [kh][kw][Cout][Cin] (K-major B operand of the forward GEMM);  w_t_lo / w_lo =
 * the low parts w - tf32_trunc(w) in the transposed / the HWIO order (SE_MODE_TF32X3).  se_split_filters writes all
 * three for every kernel of a flat parameter buffer in one launch. */
typedef struct {
  const float* w_t;
  const float* w_t_lo;
  const float* w_lo;
} se_conv_aux;
int se_conv2d_fwd_aux(const se_conv_desc* d, const float* x, const float* w, const se_conv_aux* aux, const float* bias,
                      const float* residual, float* y, int relu, double* stats, int mode, void* stream);
int se_conv2d_dgrad_aux(const se_conv_desc* d, const float* dy, const float* w, const se_conv_aux* aux, float* dx, float beta,
                        int mode, void* stream);
/* se_transpose_filters + PL[off + i] = lo(P[off + i]), PTL[off + (tap, co, ci)] = lo(P[off + (tap, ci, co)]) */
int se_split_filters(const float* P, float* PT, float* PL, float* PTL, const int64_t* table, int n, void* stream);
/* PT[off + (tap, co, ci)] = P[off + (tap, ci, co)] for n kernels of a flat buffer, one launch.
 * table: host array of n x {element offset, taps, Cin, Cout} (int64). */
int se_transpose_filters(const float* P, float* PT, const int64_t* table, int n, void* stream);
/* dx = beta*dx + conv^T(dy, w)   (gradient wrt the input; autodiff of the above) */
int se_conv2d_dgrad(const se_conv_desc* d, const float* dy, const float* w, float* dx, float beta,
                    int mode, void* stream);
/* dw += x (*) dy ; dbias += sum_pixels dy   (dbias may be NULL). Accumulates: caller zeroes.
 * Split-K partial sums go through a workspace of the library, one per device and stream (se_init prepares the one of
 * se_run_ops' side stream), and are added in a fixed order: the same result on every run.  When a request does not fit
 * the 32 MB workspace, or a stream's first call is inside a graph capture, the partial sums are added with atomics
 * instead (same values up to the order of float additions). */
int se_conv2d_wgrad(const se_conv_desc* d, const float* x, const float* dy, float* dw, float* dbias,
                    int mode, void* stream);
/* Which kernel family takes this layer in `mode` (pure host-side planning: no device work, callable without a GPU):
 * 1 = a tensor-core kernel, 0 = an fp32 kernel; direction 0 forward, 1 backward data, 2 weight gradient.  (Forward: given the
 * auxiliary kernel copies of se_conv_aux; with BatchNorm statistics wider than 384 channels the sums come from a separate
 * se_bn_stats pass, see se_conv2d_fwd_aux.)  The plan sees the descriptor only, not the buffers: a weight gradient whose
 * dw or dbias is not 16-byte aligned runs on the fp32 kernels even where this returns 1. */
int se_conv2d_path(const se_conv_desc* d, int mode, int direction);
/* Dense (models/cifar_resnet.py:233, plainnet.py:67,76, wide_residual_network.py:96, utils.py:242,
 * learn_image_embeddings.py:44): y = x W + b as a 1x1 convolution over a (B,1,1,Cin) tensor. */
int se_dense_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Cin, int Cout,
                 int relu, double* stats, int mode, void* stream);
int se_dense_bwd(const float* x, const float* w, const float* dy, float* dx, float beta, float* dw,
                 float* dbias, int B, int Cin, int Cout, int mode, void* stream);

/* ------------------------------------------------------------------ batch normalisation
 * keras.layers.BatchNormalization (cifar_resnet.py:100,107,220; plainnet.py:53,68,71;
 * wide_residual_network.py:14,25,44,51,91; learn_image_embeddings.py:43), fused with the
 * Activation('relu') / layers.add / AveragePooling2D+ChannelPadding shortcut that follow it
 * (cifar_resnet.py:101,117-124). rows = N*H*W. */
typedef struct {
  const float* ptr;       /* NULL = no residual */
  int32_t C;              /* channels of the residual tensor (<= C of the BN output) */
  int32_t pad_lo;         /* ChannelPadding: residual channel c lands on output channel c+pad_lo */
  int32_t pool;           /* 1 = same resolution, 2 = 2x2 average pool of a (N,2H,2W,C) tensor */
  int32_t H, W;           /* spatial size of the BN output (needed when pool == 2) */
} se_residual;

/* accumulate sum(x), sum(x^2) per channel into stats (float64 [2C], caller zeroes) */
int se_bn_stats(const float* x, int64_t rows, int C, double* stats, void* stream);
/* training mode: mean/var (biased) from `stats`; y = relu?( gamma*(x-mean)*rsqrt(var+eps)+beta + res );
 * writes save_mean/save_invstd [C] for the backward pass and updates moving statistics
 * (moving = moving*momentum + batch*(1-momentum); variance fed as var*n/(n-(1+eps))). */
int se_bn_fwd_train(const float* x, int64_t rows, int C, const double* stats, const float* gamma,
                    const float* beta, float eps, float momentum, float* moving_mean, float* moving_var,
                    float* save_mean, float* save_invstd, const se_residual* res, int relu, float* y,
                    void* stream);
/* Conv2D followed by training-mode BatchNormalization (+ same-shape residual, + ReLU): the pair the reference stacks in
 * every block (models/cifar_resnet.py:96-107, models/wide_residual_network.py:28-66, models/plainnet.py), as ONE call:
 *   y      = conv(x, w) [+ bias] [relu]                (kept: the BatchNorm backward needs it)
 *   bn_out = act( gamma*(y-mean)*rsqrt(var+eps)+beta [+ res] ), statistics / moving averages as se_bn_fwd_train
 * = se_conv2d_fwd_ex (statistics accumulated in the convolution epilogue) + se_bn_fwd_train.  (Round 1 also had a
 * single-launch form with a grid barrier inside the convolution kernel; measured 0.13 ms per step SLOWER than the two
 * launches, it was removed in round 2.)  stats: float64 [2*Cout], caller zeroes; `counter` is unused. */
int se_conv_bn_fwd(const se_conv_desc* d, const float* x, const float* w, const float* w_t, const float* bias,
                   float* y, int relu, double* stats, const float* gamma, const float* beta, float eps, float momentum,
                   float* moving_mean, float* moving_var, float* save_mean, float* save_invstd, const float* res,
                   int bn_relu, float* bn_out, void* counter, int mode, void* stream);
/* inference mode (learn_image_embeddings.py:271 predict_generator): moving statistics */
int se_bn_fwd_infer(const float* x, int64_t rows, int C, const float* gamma, const float* beta,
                    const float* moving_mean, const float* moving_var, float eps, const se_residual* res,
                    int relu, float* y, void* stream);
/* backward of se_bn_fwd_train.  dout = gradient wrt y; `y` is needed when relu != 0 (mask y > 0).
 *   g  = dout * (y > 0)                                  (relu)          [also the residual gradient]
 *   dgamma += sum g*xhat ; dbeta += sum g                 (accumulate: caller zeroes)
 *   dx = beta_dx*dx + gamma*invstd*(g - mean(g) - xhat*mean(g*xhat)) [* (x > 0) if relu_in]
 *   dres = beta_res*dres + g      (same-resolution residual only; NULL to skip)
 * scratch: float64 [2C + 1] (sums + the arrival counter of the fused single-launch path), caller zeroes.
 * relu_in: x itself is a relu output (plainnet.py:52-53). */
int se_bn_bwd(const float* x, const float* y, const float* dout, int64_t rows, int C, const float* gamma,
              const float* save_mean, const float* save_invstd, int relu, int relu_in, float* dx,
              float beta_dx, float* dres, float beta_res, float* dgamma, float* dbeta, double* scratch,
              void* stream);
/* Which implementation se_bn_bwd runs for (rows, C) on a device with `sms` SMs (sms <= 0: the current device; a positive
 * sms is pure host-side planning, callable without a GPU).  se_bn_bwd decides by the same function, and SE_BN_NO_FUSE /
 * SE_BN_NO_REG in the environment move both alike.  Bits 0-1 name the path, bit 2 its float4 / fixed-quad variant:
 *   SE_BN_BWD_SCALAR       bn_bwd_reduce_kernel + bn_bwd_apply_kernel, scalar branch (C % 4 != 0)          2 launches
 *   SE_BN_BWD_VEC          the same two kernels, float4 branch                                             2 launches
 *   SE_BN_BWD_SLAB_ATOMIC  bn_bwd_fused_kernel (slab in shared memory, grid barrier), per-element shared
 *                          atomics: 512 threads do not divide into channel quads (512 % (C/4) != 0)        1 launch
 *   SE_BN_BWD_SLAB_QUAD    bn_bwd_fused_kernel, every thread keeps one channel quad                         1 launch
 *   SE_BN_BWD_SLAB_REG     bn_bwd_reg_kernel (slab in registers, grid barrier): C <= 128, 512 % (C/4) == 0,
 *                          at most 8 float4 of the slab per thread                                          1 launch
 * The slab paths hold rows/sms rows per CTA (rounded up to a multiple of 4) and need them to fit; every
 * other C % 4 == 0 layer is SE_BN_BWD_VEC.  Returns < 0 (SE_ERR_ARG) for rows <= 0 or C <= 0. */
#define SE_BN_BWD_SCALAR 0
#define SE_BN_BWD_SLAB_ATOMIC 1
#define SE_BN_BWD_SLAB_REG 2
#define SE_BN_BWD_VEC 4
#define SE_BN_BWD_SLAB_QUAD 5
int se_bn_bwd_path(int64_t rows, int C, int sms);
/* gradient of the pooled / channel-padded shortcut (cifar_resnet.py:117-121):
 * dsrc[n,2h+i,2w+j,c] = beta*dsrc + 0.25 * g[n,h,w,c+pad_lo], g = dout*(y>0) if relu. */
int se_shortcut_bwd(const float* dout, const float* y, int relu, int N, int H, int W, int C,
                    const se_residual* res, float* dsrc, float beta, void* stream);

/* ------------------------------------------------------------------ pooling / elementwise */
int se_avgpool2_fwd(const float* x, float* y, int N, int H, int W, int C, void* stream);       /* plainnet.py:59 */
int se_avgpool2_bwd(const float* dy, float* dx, float beta, int N, int H, int W, int C, void* stream);
int se_maxpool_fwd(const float* x, float* y, int N, int H, int W, int C, int k, int stride, int pad_t,
                   int pad_l, int Ho, int Wo, void* stream);                                    /* ResNet-50 pool1 */
int se_maxpool_bwd(const float* x, const float* y, const float* dy, float* dx, int N, int H, int W, int C,
                   int k, int stride, int pad_t, int pad_l, int Ho, int Wo, void* stream);
int se_gap_fwd(const float* x, float* y, int N, int HW, int C, void* stream);                  /* cifar_resnet.py:228 */
int se_gap_bwd(const float* dy, float* dx, float beta, int N, int HW, int C, void* stream);
/* y = a + b [relu]; backward: da = beta*da + g, db likewise, g = dy*(y>0)  (wide_residual_network.py:34,56) */
int se_add_fwd(const float* a, const float* b, float* y, int64_t n, int relu, void* stream);
int se_add_bwd(const float* dy, const float* y, int relu, float* da, float beta_a, float* db, float beta_b,
               int64_t n, void* stream);
/* y = relu(x) ; dx = beta*dx + dy*(y>0)  (learn_image_embeddings.py:42) */
int se_relu_fwd(const float* x, float* y, int64_t n, void* stream);
int se_relu_bwd(const float* dy, const float* y, float* dx, float beta, int64_t n, void* stream);

/* ------------------------------------------------------------------ embedding head (north-star item)
 * One fused kernel for utils.l2norm (utils.py:125-127), the target gather E[y]
 * (learn_image_embeddings.py:48-50), utils.inv_correlation / squared_distance (utils.py:34-46),
 * the metric utils.nn_accuracy (utils.py:57-100, k<=1) and the backward pass of all of it.
 *   z [B,ldz] raw network output; E [C,ldE] class matrix (fp32); labels int32 [B]
 *   x_out [B,ldz]  = wrapped output (l2norm(z) for INV_CORR, z otherwise)   (may be NULL)
 *   loss [B], acc [B] per-sample loss and 0/1 accuracy                       (may be NULL)
 *   dz [B,ldz]     = d( loss_scale * sum_b loss_b )/dz + Jx^T extra_dx, where extra_dx [B,ldz]
 *                    (may be NULL) is a gradient wrt x_out coming from the classifier branch
 *                    (learn_image_embeddings.py:34-44, --cls_weight)        (dz may be NULL)
 * loss_scale is 1/global_batch for Keras' mean-over-batch. */
int se_embed_head_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B,
                          int D, int C, int loss_kind, float loss_scale, const float* extra_dx,
                          float* x_out, float* loss, float* acc, float* dz, void* stream);
/* same + rank_out [B] (may be NULL): the top-k form of the metric for every k at once.  utils.nn_accuracy(k)
 * (utils.py:85,95) is 1 iff one of the k best class scores lies within 1e-6 of the true class' score; with G = number
 * of classes better than the true score by >= 1e-6, that is `rank_out < k` (rank_out = G, or C when no class is within
 * 1e-6).  For SE_LOSS_SOFTMAX_CORR (metric = Keras categorical / top-k categorical accuracy) rank_out = number of
 * outputs strictly above the output at argmax(t).  --top_k_acc K: accuracy@K = mean(rank_out < K). */
int se_embed_head_fwd_bwd_ex(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B,
                             int D, int C, int loss_kind, float loss_scale, const float* extra_dx,
                             float* x_out, float* loss, float* acc, float* dz, float* rank_out, void* stream);
/* the DeViSE hinge ranking loss (utils.devise_ranking_loss, learn_devise.py) with the same arguments plus the margin m;
 * loss_kind must be SE_LOSS_DEVISE_RANK (se_embed_head_fwd_bwd_ex rejects it).  No output wrapper: x_out = z.
 *   loss[b] = sum_c relu(m - <t,z> + <z,E_c>) - m             (t = E[label])
 *   dz      = loss_scale * (sum_{c in A} E_c - |A| t) + extra_dx,  A = {c : m - <t,z> + <z,E_c> > 0} (strict)
 *   acc, rank_out: those of SE_LOSS_UNNORM_CORR (max_sim_acc), bit for bit
 * The gradient sums the active rows in class order: reruns give the same bits. */
int se_devise_rank_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* E, int ldE, int B, int D, int C,
                           int loss_kind, float loss_scale, const float* extra_dx, float* x_out, float* loss, float* acc,
                           float* dz, float* rank_out, float margin, void* stream);
/* softmax + Keras categorical_crossentropy (clip 1e-7) + argmax accuracy + backward
 * (learn_image_embeddings.py:44,230-231): dlogits = scale * dCE/dlogits. */
int se_softmax_xent_fwd_bwd(const float* logits, int ld, const int32_t* labels, int B, int C, float scale,
                            float* prob, float* loss, float* acc, float* dlogits, void* stream);
/* same + rank_out [B] (may be NULL): classes with a strictly larger logit than the label's -- utils.top_k_acc(k)
 * (utils.py:49-54, in_top_k) = mean(rank_out < k) */
int se_softmax_xent_fwd_bwd_ex(const float* logits, int ld, const int32_t* labels, int B, int C, float scale,
                               float* prob, float* loss, float* acc, float* dlogits, float* rank_out, void* stream);
/* the same with label smoothing (learn_classifier.py:17-22 transform_inputs + Keras categorical_crossentropy): for
 * 0 < smoothing < 1 the targets are t_hi = float(1 - smoothing) on the label and t_lo = float(smoothing / (C - 1)) on
 * every other class (C >= 2); any other value means one-hot targets and runs se_softmax_xent_fwd_bwd_ex.
 *   loss[b]    = -sum_c t_c log clip(p_c, 1e-7, 1 - 1e-7), over all classes
 *   dlogits    = scale * (p_j T - live_j t_j), live = 1e-7 <= p <= 1 - 1e-7 (tf.clip_by_value's gradient mask),
 *                T = sum_c live_c t_c
 *   acc, rank_out: as above against argmax(y_true) -- the label, or the lowest other index when t_lo > t_hi
 *                (smoothing > (C-1)/C) */
int se_softmax_xent_smooth_fwd_bwd(const float* logits, int ld, const int32_t* labels, int B, int C, float smoothing,
                                   float scale, float* prob, float* loss, float* acc, float* dlogits, float* rank_out,
                                   void* stream);
/* the loss of the label embedding network (Sun et al.; learn_labelembedding.py:21-37) and its gradients.  out1, out2
 * [B, ld] are the logits of 'prob' and 'out2', emb [C, ldE] the label-embedding table, tar = emb[y].  With
 * p1 = softmax(out1), p2 = softmax(out2), q2 = softmax(out2 / tau), s = softmax(tar) and Keras' sparse cross-entropy on
 * probabilities, sCE(p, y) = -log c_y + log sum_j c_j with c = clip(p, 1e-7, 1 - 1e-7) (gradient only where the clip is
 * inactive):
 *   mask_i   = argmax(out2_i) == y_i (first maximum)        F = B_eff / (sum_i mask_i + 1e-8)   (float32)
 *   loss[i]  = beta sCE(p1, y) - (1-beta) sum_j s_j log_softmax(out1)_j + sCE(p2, y)
 *              - sum_j q2_j log_softmax(tar)_j * mask_i * F + relu(p2_y - alpha)
 *   acc[i]   = argmax(out1_i) == y_i (first maximum)
 *   d_out1   = scale * (beta dsCE(p1, y)/dout1 + (1-beta) (p1 sum_j s_j - s))
 *   d_out2   = scale * (dsCE(p2, y)/dout2 + [p2_y > alpha] p2_y (e_y - p2))      (q2, s and mask carry no gradient)
 *   d_emb[c] = scale * F * sum_{i: y_i = c, mask_i} (s_i sum_j q2_ij - q2_i)   summed in increasing i; every row of
 *              d_emb [C, ldE] is written (zeros for classes without such a sample)
 * Rows with a label outside [0, C) (label < 0: padding) count neither in B_eff nor in sum mask; their loss, accuracy
 * and gradients are 0.  B_eff is the number of the other rows.  loss, acc, d_out1, d_out2 and d_emb may be NULL.
 * work: se_labelembed_workspace_bytes(B, C) bytes, 16-byte aligned; it starts with [B] float4
 * {mask, CE(q2, softmax(tar)), beta sCE(p1) + (1-beta) CE(s, p1) + sCE(p2), relu term}.  1 <= B <= 8192, C >= 2,
 * tau > 0; else SE_ERR_ARG.  Two launches, no float atomics: reruns give the same bits. */
int64_t se_labelembed_workspace_bytes(int B, int C);
int se_labelembed_fwd_bwd(const float* out1, const float* out2, int ld, const int32_t* labels, const float* emb, int ldE,
                          int B, int C, float tau, float alpha, float beta, float scale, float* loss, float* acc,
                          float* d_out1, float* d_out2, float* d_emb, void* work, void* stream);
/* the center loss of Wen et al. (learn_center_loss.py:17-41) and its gradients.  z [B, ldz] is the raw embedding,
 * cent [C, ldc] the class centroids (the 'cls_centroids' Embedding), labels [B] the classes.  For every row b with
 * 0 <= y_b < C, d_b = z_b - cent[y_b]:
 *   loss[b]    = 1/2 sum_j d_bj^2                                  (the unweighted per-sample center loss)
 *   d_z[b]     = scale * d_b                                       (overwritten, not accumulated)
 *   d_cent[k]  = -scale * sum_{b: y_b = k} (z_b - cent[k])         summed in increasing b; every row k of d_cent [C, ldc]
 *                is written (zeros for a class without a sample)
 * scale is the loss weight over the global batch (w / (B * world) for Keras' mean).  Rows with a label outside [0, C)
 * (padding) get loss 0 and d_z 0 and take no part in d_cent.  Only the first D columns of every row are read or
 * written.  loss, d_z and d_cent may each be NULL (skipped).  B, C, D >= 1, ldz >= D, ldc >= D, z, labels and cent not
 * NULL; else SE_ERR_ARG.  One launch, no float atomics: reruns give the same bits. */
int se_center_loss_fwd_bwd(const float* z, int ldz, const int32_t* labels, const float* cent, int ldc, int B, int C, int D,
                           float scale, float* loss, float* d_z, float* d_cent, void* stream);

/* ------------------------------------------------------------------ optimizer
 * keras.optimizers.SGD(lr, momentum, decay, nesterov, clipnorm) + kernel_regularizer=l2(.)
 * (learn_image_embeddings.py:229-236; cifar_resnet.py:152; plainnet.py:8) over ONE flat fp32
 * parameter / gradient / velocity buffer.  Segments give the L2 coefficient of a range.
 *   pass 1: g += 2*lambda*p on regularised ranges; out[0] = sum g^2, out[1] = sum lambda*p^2
 *   pass 2: scale = clipnorm/norm if norm >= clipnorm; v = m*v - lr*g*scale; p += v
 *           (nesterov: p += m*v - lr*g*scale)
 * `out` is float64[2] device memory (caller zeroes before pass 1). */
typedef struct {
  int64_t begin, end;     /* element range [begin,end) of the flat buffer */
  float l2;               /* lambda */
} se_l2_segment;
int se_sgd_step(float* p, float* g, float* v, int64_t n, const se_l2_segment* segs, int nsegs, float lr,
                float momentum, int nesterov, float clipnorm, double* out, void* stream);
/* the two passes separately (data-parallel runs all-reduce g between nothing and pass 1) */
int se_sgd_prepare(const float* p, float* g, int64_t n, const se_l2_segment* segs, int nsegs, double* out,
                   void* stream);
int se_sgd_apply(float* p, const float* g, float* v, int64_t n, float lr, float momentum, int nesterov,
                 float clipnorm, const double* out, void* stream);

/* Keras SGD(decay) (learn_image_embeddings.py:224-236, --max_decay): lr_state = float[4] device memory
 * {lr written by the schedule, decay, iterations, lr_t}; one call per optimizer step sets lr_t = lr / (1 + decay *
 * iterations) and increments iterations.  se_sgd_apply_devlr then reads lr_state + 3. */
int se_sgd_schedule(float* lr_state, void* stream);
/* same as se_sgd_apply with the learning rate read from device memory (float[1]) at run time, so
 * that a CUDA-graph-captured step follows the SGDR schedule (sgdr_callback.py:75-87) without re-capture */
int se_sgd_apply_devlr(float* p, const float* g, float* v, int64_t n, const float* lr_dev, float momentum,
                       int nesterov, float clipnorm, const double* out, void* stream);
/* keras.optimizers.Adagrad(lr, epsilon, decay) (learn_devise.py:87,114), the update pass after se_sgd_prepare: with
 * s = clipnorm/norm when clipnorm > 0 and norm = sqrt(out[0]) >= clipnorm, else 1, per element
 *   a += (s g)^2 ;  p -= lr_t s g / (sqrt(a) + epsilon)
 * a [n] is the accumulator (zero at the start of a training phase); lr_dev is the lr_t of se_sgd_schedule (lr_state + 3). */
int se_adagrad_apply_devlr(float* p, const float* g, float* a, int64_t n, const float* lr_dev, float epsilon, float clipnorm,
                           const double* out, void* stream);

/* ------------------------------------------------------------------ data-parallel gradient exchange
 * keras.utils.multi_gpu_model (learn_image_embeddings.py:133,148) -> one process per GPU + NCCL.  The communicator lives
 * inside the library so that the plan runner can issue bucketed all-reduces on its own stream while the backward pass
 * continues and capture them in the step's CUDA graph (SE_OP_ALLREDUCE in se_run_ops).  NCCL is taken from the
 * libnccl.so.2 already loaded in the process; SE_ERR_UNSUPPORTED when there is none.
 *   se_comm_unique_id: rank 0 creates the 128-byte NCCL id, the caller distributes it (any out-of-band channel);
 *   se_comm_init:      collective over all ranks, current CUDA device = this rank's GPU;
 *   se_allreduce_sum:  in-place SUM over all ranks of buf[0:n] on `stream` (per-sample losses are pre-scaled by
 *                      1/global_batch, so the sum IS the gradient of the global mean loss). */
int se_comm_unique_id(void* id_out, int bytes);
int se_comm_init(int rank, int world, const void* unique_id, int bytes);
int se_comm_world(void);
int se_allreduce_sum(float* buf, int64_t n, void* stream);
int se_comm_destroy(void);

/* ------------------------------------------------------------------ input pipeline
 * TinyDatasetGenerator.compose_batch (datasets/common.py:771-796): Keras ImageDataGenerator.random_transform with
 * horizontal_flip + width/height_shift_range 0.15 (datasets/common.py:640; shift = scipy affine_transform order 1,
 * mode 'nearest') and .standardize (featurewise mean / std, :639) for a batch gathered by index from a dataset that is
 * resident in device memory.  src [n, H, W, C] uint8 or float32 raw pixels; index [B] rows of src (NULL = 0..B-1);
 * tx / ty [B] row / column shifts in pixels (NULL = 0), flip [B] 0/1 (NULL = none) -- the random draws are the host's;
 * mean / inv_std [C] with inv_std = 1 / (std + 1e-7); out [B, H, W, C] float32. */
int se_augment_batch(const void* src, int src_is_u8, const int32_t* index, const float* tx, const float* ty,
                     const unsigned char* flip, const float* mean, const float* inv_std, float* out, int B, int H, int W,
                     int C, void* stream);

/* File datasets (NABirds / CUB): FileDatasetGenerator.compose_batch (datasets/common.py:380-432) after the decode, for a
 * batch of B images decoded on the host to uint8 RGB (HWC) and packed into one device buffer `src`.  Per image, one
 * descriptor (desc_host for the checks and the launch plan, desc_dev the same array in device memory for the kernel):
 *   src_offset    byte offset of the image in src; src_h x src_w its size (each side <= SE_RESAMPLE_MAX_SIDE)
 *   rh x rw       the size PIL resize(BILINEAR) gives it (>= the crop, <= SE_RESAMPLE_MAX_RESIZED; source / resized
 *                 <= 31 on each axis) -- resampled bit-exactly like Pillow's libImaging/Resample.c, see file_augment.cu
 *   flip          1: the resized image is mirrored left-right before the erase and the crop
 *   ey, ex, eh, ew  erase rectangle in the (flipped) resized image, eh = 0: none
 *   cy, cx        crop offset in the (flipped) resized image; the crop is crop_h x crop_w (<= SE_RESAMPLE_MAX_CROP)
 *   noise_id      the image's number in the erase noise (its position in the global batch; 0 <= noise_id < 2^20)
 * out [B, crop_h, crop_w, 3] float32 = (x - mean[c]) / std[c] (float32 subtraction, IEEE division, no epsilon), with the
 * channels reversed when bgr = 1 (normalised in RGB order first, datasets/common.py:514-520).  An erased pixel holds
 * (float)((u - (double)mean[c]) / (double)std[c]) with mean / std in RGB order even when bgr = 1 (as :538-540) and
 *   u = se_erase_noise(seed, b, y, x, c), b = noise_id, (y, x) the pixel in the flipped resized image, c the output channel:
 *     z = seed + (((((b << 20) | y) << 20 | x) << 2 | c) + 1) * 0x9E3779B97F4A7C15     (uint64, wrapping)
 *     z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9;  z = (z ^ (z >> 27)) * 0x94D049BB133111EB;  z ^= z >> 31
 *     u = (double)(z >> 11) * 2^-53 * 255.0                                         (in [0, 255))
 * mean / std are host arrays of 3.  SE_ERR_ARG for any descriptor outside these limits (there is no reflect padding),
 * and when a crop row's tables, 4 * crop_w * (3 * 8 + taps + 2) bytes, leave no room for a band row in 200 KB of shared
 * memory (taps = 2 * ceil(source / resized) + 1 on the horizontal axis).
 * One launch, no atomics: reruns give the same bits. */
#define SE_RESAMPLE_MAX_SIDE 4096
#define SE_RESAMPLE_MAX_RESIZED 65535
#define SE_RESAMPLE_MAX_CROP 1024
typedef struct {
  int64_t src_offset;
  int32_t src_h, src_w, rh, rw;
  int32_t flip, ey, ex, eh, ew;
  int32_t cy, cx, noise_id;
} se_resample_desc;
int se_resample_crop_batch(const unsigned char* src, const se_resample_desc* desc_host, const se_resample_desc* desc_dev,
                           int B, int crop_h, int crop_w, const float* mean, const float* std, int bgr, uint64_t seed,
                           float* out, void* stream);

/* JPEG decoding for the file datasets, bit-identical to what Pillow (libjpeg-turbo, default settings: integer IDCT,
 * fancy upsampling) returns after convert('RGB'); see jpeg_parse.cu and jpeg_decode.cu.
 *
 * se_jpeg_parse (host, no device needed) walks the markers of one file of n bytes -- never reading past n -- and fills
 * *out.  It returns out->status: SE_JPEG_OK when the device can decode the file, else the reason it cannot (the file
 * then takes the host decoder).  Supported: 8-bit baseline / extended sequential Huffman (SOF0 / SOF1) in one scan, 1
 * component, or 3 components that libjpeg reads as YCbCr (its jdapimin.c rule: JFIF marker, else the Adobe transform
 * flag, else the component ids) with luma sampling h, v in {1, 2} and chroma 1x1, sides <= SE_RESAMPLE_MAX_SIDE, and a
 * well-formed restart marker sequence.  SE_ERR_ARG for null pointers or n < 0.
 * se_jpeg_pack (host) writes the scan of a supported file into `out` (cap >= out->packed_bytes) without byte stuffing
 * and restart markers:  uint32 int_start[n_intervals + 1] (byte offset of each restart interval in the data, then its
 * size), uint32 sub_first[n_intervals + 1] (first subsequence of each interval), zero padding to 16 bytes, the data,
 * 16 zero bytes.  An interval of L bytes is cut into max(1, ceil(L / SE_JPEG_SUBSEQ_BYTES)) subsequences.  Returns the
 * bytes written, or < 0.
 * se_jpeg_workspace_bytes (host) sets job[i].ws_offset for a batch of B supported images and returns the device
 * workspace the batch needs (< 0 on bad arguments).
 * se_jpeg_decode_batch decodes the batch into `out`: image i, described by info_host[i] (host) and the same bytes at
 * in + job[i].info_offset (device), with its se_jpeg_pack output at in + job[i].packed_offset, becomes H x W x 3 uint8
 * RGB at out + job[i].out_offset.  job_host / job_dev: the same jobs in host and device memory.  status[i] (device) is
 * set to SE_JPEG_OK, or to SE_JPEG_DEV_CORRUPT when the entropy-coded data ends, or holds a code no table matches,
 * before the image's last block, or a dequantised coefficient falls outside int16 (where libjpeg-turbo's SIMD and C
 * paths differ); the pixels of such an image are undefined.  Quantisation values above 32767 are SE_JPEG_MALFORMED.
 * Three plain launches (not programmatic dependent ones) and a memset of the workspace; no
 * atomics on data: reruns give the same bits. */
#define SE_JPEG_OK 0
#define SE_JPEG_NOT_JPEG 1        /* no SOI marker */
#define SE_JPEG_TRUNCATED 2       /* the file ends inside a segment or the scan, or before EOI */
#define SE_JPEG_MALFORMED 3       /* a segment or table libjpeg would reject or warn about */
#define SE_JPEG_PROGRESSIVE 4     /* SOF2 / SOF6 */
#define SE_JPEG_ARITHMETIC 5      /* SOF9 - SOF15 arithmetic coding, DAC */
#define SE_JPEG_OTHER_PROCESS 6   /* lossless or hierarchical (SOF3, SOF5 - SOF7) */
#define SE_JPEG_PRECISION 7       /* not 8-bit samples */
#define SE_JPEG_COMPONENTS 8      /* neither 1 nor 3 components (CMYK, YCCK, ...) */
#define SE_JPEG_COLORSPACE 9      /* 3 components libjpeg does not read as YCbCr (RGB) */
#define SE_JPEG_SAMPLING 10       /* sampling other than 4:4:4, 4:2:2, 4:2:0, 4:4:0 */
#define SE_JPEG_MULTISCAN 11      /* more than one scan, or a scan without every component */
#define SE_JPEG_SIZE 12           /* a side of 0 (DNL) or above SE_RESAMPLE_MAX_SIDE */
#define SE_JPEG_RESTART 13        /* restart markers out of sequence, or not the interval count */
#define SE_JPEG_NUM_REASONS 14
#define SE_JPEG_DEV_CORRUPT 1     /* device status word */
#define SE_JPEG_SUBSEQ_BYTES 128
typedef struct {
  uint16_t lookup[512];   /* next 9 bits of the stream -> (code length << 8) | symbol; 0: the code is longer */
  int32_t maxcode[18];    /* largest code of length l (index l = 1..16), -1 when there is none */
  int32_t valoffset[18];  /* huffval index of a code of length l = code + valoffset[l] */
  uint8_t huffval[256];
} se_jpeg_huff;
typedef struct {
  int32_t status;                         /* SE_JPEG_OK or the reason the device does not decode the file */
  int32_t width, height;
  int32_t ncomp;                          /* 1 or 3 */
  int32_t comp_id[3], h[3], v[3], tq[3];  /* per component: id, sampling factors, quantisation table */
  int32_t td[3], ta[3];                   /* per component: DC / AC Huffman table of the scan */
  int32_t hmax, vmax;
  int32_t mcus_x, mcus_y;                 /* MCUs per row / column (blocks, for a 1-component scan) */
  int32_t restart_interval;               /* MCUs per restart interval, 0: none */
  int32_t n_intervals, n_subseq;
  int32_t saw_jfif, saw_adobe, adobe_transform;
  int32_t qt_mask;                        /* bit t: quantisation table t was defined */
  int32_t reserved;
  int64_t scan_begin, scan_end;           /* the entropy-coded segment, RST markers included: bytes [begin, end) */
  int64_t data_bytes;                     /* its size without byte stuffing and markers */
  int64_t packed_bytes;                   /* size of the se_jpeg_pack output */
  uint16_t qt[4][64];                     /* quantisation tables in natural (row-major) order */
  se_jpeg_huff dc[4], ac[4];
} se_jpeg_info;
typedef struct {
  int64_t info_offset;    /* se_jpeg_info of the image in `in` (8-byte aligned) */
  int64_t packed_offset;  /* its se_jpeg_pack output in `in` (16-byte aligned) */
  int64_t out_offset;     /* its RGB output in `out` */
  int64_t ws_offset;      /* its part of the workspace (set by se_jpeg_workspace_bytes) */
} se_jpeg_job;
int se_jpeg_parse(const uint8_t* data, int64_t n, se_jpeg_info* out);
int64_t se_jpeg_pack(const uint8_t* data, int64_t n, const se_jpeg_info* info, uint8_t* out, int64_t cap);
int64_t se_jpeg_workspace_bytes(const se_jpeg_info* info, se_jpeg_job* job, int B);
int se_jpeg_decode_batch(const unsigned char* in, const se_jpeg_info* info_host, const se_jpeg_job* job_host,
                         const se_jpeg_job* job_dev, int B, unsigned char* out, int32_t* status, void* workspace,
                         int64_t workspace_bytes, void* stream);
/* sizeof(se_jpeg_info), sizeof(se_jpeg_huff), sizeof(se_jpeg_job), then the offset of every field of se_jpeg_info,
 * se_jpeg_huff and se_jpeg_job in declaration order (for bindings to check their mirrors); returns the count written
 * (at most cap), or the count needed when out is NULL. */
int se_jpeg_layout(int64_t* out, int cap);

/* ------------------------------------------------------------------ retrieval
 * evaluate_retrieval.py:56-63: rows [row0,row0+rows) of the N x N distance matrix of F [N,ldF]
 * (fp32, D columns) against all N columns; out [rows, ldout].  normalize=1 applies line 58
 * (F /= ||F||) on the fly without mutating F.  `workspace` (device, >= se_pairwise_workspace_bytes)
 * holds the row norms and, for the tensor-core path, the split operands. */
int64_t se_pairwise_workspace_bytes(int N, int D, int mode);
int se_pairwise_dist(const float* F, int ldF, int N, int D, int row0, int rows, int pdist_mode,
                     int normalize, float* out, int64_t ldout, void* workspace, int mode, void* stream);

/* Fused distance + ranking (SURVEY.md section 8(f) rank 1): the k nearest items (ascending distance, ties by index) of
 * query rows [row0, row0+rows) WITHOUT writing the rows x N distance matrix -- sample-based per-row thresholds, a
 * tensor-core sweep that keeps only the entries below them, a per-row sort of those candidates.  Distances are the
 * ones se_pairwise_dist would store (same arithmetic), so out_idx equals se_row_topk of that matrix.
 * status [1] device int32: 0 = exact; non-zero = some row found fewer than k or more than 4096 candidates (pathological
 * distance distributions) and the caller must use se_pairwise_dist + se_row_topk instead.  k <= 1024, D <= 128.
 * out_idx [rows, ldo] int32, out_val [rows, ldo] float32 (may be NULL). */
int64_t se_pairwise_topk_workspace_bytes(int N, int D, int rows);
int se_pairwise_topk(const float* F, int ldF, int N, int D, int row0, int rows, int pdist_mode, int normalize, int k,
                     int32_t* out_idx, float* out_val, int ldo, void* workspace, int32_t* status, void* stream);

/* Ranking step of evaluate_retrieval.py:67 (`np.argsort(pdist, axis=-1)`) restricted to what the metrics read
 * (class_hierarchy.py:242-244,273,283: the first clip_ahp+1 ranks): for each of `rows` rows of dist [rows, ld] the k
 * smallest of its n values in ascending order, ties by ascending index (a stable argsort's prefix; -0.0 == +0.0).
 * out_idx [rows, ldo] int32 column indices, out_val [rows, ldo] the distances (may be NULL).  k <= 1024 and
 * n <= ~52000 (a row is staged in shared memory), else SE_ERR_UNSUPPORTED. */
int se_row_topk(const float* dist, int64_t ld, int rows, int n, int k, float* out_val, int32_t* out_idx, int ldo,
                void* stream);

/* ClassHierarchy.hierarchical_precision(retrieved, labels, ks, compute_ahp=clip, ignore_qids=True) of the reference
 * (class_hierarchy.py:211-316) on the first K1 = max(ks, clip) + 1 ranks of Q queries (query ids q0 .. q0+Q-1 are
 * database indices; ranks [Q, ldr] int32, e.g. from se_row_topk).  labels [N] int32 class indices (< C);
 * wup_lut / lcs_height_lut [C, C] float64 = wup_similarity / lcs_height of the hierarchy; best_wup / best_lcs [C, K1]
 * float64 = per query class the cumulative sums of the descending class similarities of the WHOLE database
 * (ranking independent, class_hierarchy.py:268,280).  out [Q, 2*(nks + (clip > 0))] float64 per query:
 * P@ks[0] (WUP), P@ks[0] (LCS_HEIGHT), ..., AHP@clip (WUP), AHP@clip (LCS_HEIGHT).  nks <= 8. */
int se_hier_precision(const int32_t* ranks, int ldr, int Q, int K1, int q0, const int32_t* labels, int C,
                      const double* wup_lut, const double* lcs_height_lut, const double* best_wup, const double* best_lcs,
                      const int32_t* ks, int nks, int clip, double* out, void* stream);

/* The same metrics from rankings of any length, as evaluate_retrieval.py:195 requests them (ks = 1..plot_max, compute_ahp
 * = clip or True, compute_ap = True):  ranks [Q, ldr] int32 with n_ret entries per query (n_ret = N for full rankings
 * from se_row_argsort, or max(kcurve, clip) + 1 for top-k rankings); best_wup / best_lcs [C, n_ret] float64;
 *   curve [Q, 2, kcurve] = P@k for k = 1..kcurve (WUP, LCS_HEIGHT)                       (NULL when kcurve == 0)
 *   ahp   [Q, 2]: clip > 0 -> AHP@clip, clip < 0 -> AHP over the whole list, clip == 0 -> not computed (may be NULL)
 *   ap    [Q]   : classical average precision; needs full rankings (NULL = not computed)  (class_hierarchy.py:310-314) */
int se_hier_metrics(const int32_t* ranks, int64_t ldr, int Q, int n_ret, int q0, const int32_t* labels, int C,
                    const double* wup_lut, const double* lcs_height_lut, const double* best_wup, const double* best_lcs,
                    int kcurve, int clip, double* curve, double* ahp, double* ap, void* stream);

/* Full-length ranking of evaluate_retrieval.py:67 (`np.argsort(pdist, axis=-1)`; ascending distance, ties by ascending
 * index, -0.0 == +0.0): out_idx [rows, ldo] int32 = the n column indices of every row of dist [rows, ld] in rank order.
 * workspace: se_row_argsort_workspace_bytes(rows, n) bytes of device memory (one padded row of 64-bit words per row). */
int64_t se_row_argsort_workspace_bytes(int rows, int n);
int se_row_argsort(const float* dist, int64_t ld, int rows, int n, int32_t* out_idx, int64_t ldo, void* workspace,
                   void* stream);

/* ------------------------------------------------------------------ classification (evaluate_classification_accuracy.py)
 * One-vs-rest linear SVM of the reference's train_and_predict (:20-48, sklearn LinearSVC(C): squared hinge loss, L2
 * penalty, intercept as a constant feature 1 that is regularised like the weights).  For class c, y_i = +1 where
 * labels[i] == c and -1 elsewhere, x~ = [x, 1], w~ = [W[:, c], b[c]]:
 *   f_c(w~) = 1/2 |w~|^2 + penalty * sum_i max(0, 1 - y_i w~.x~_i)^2
 * solved for all classes at once by the trust-region Newton method with conjugate-gradient steps (liblinear's primal
 * solver for L2R_L2LOSS_SVC); class c stops when |grad f_c| <= tol * max(min(pos_c, neg_c), 1) / N * |grad f_c(0)|
 * (sklearn's defaults: tol 1e-4, max_iter 1000).  The row sums are se_dense_fwd / se_dense_bwd in SE_MODE_TF32X3 with D
 * padded to a multiple of 4 and C to a multiple of 16 (zero columns); the weight gradient must add its split-K slices in
 * a fixed order, so (D+1) x C is limited by the library's workspace (about 4M elements: 2048 x 2048 fits) and
 * SE_ERR_UNSUPPORTED names the shape otherwise.  No float atomics: reruns give the same bits.
 * X [N, ldx] float32 features; labels [N] int32 in [0, C) (else SE_ERR_ARG); outputs W [D, C] (Dense layout), b [C],
 * iters [C] int32 accepted Newton steps, gnorm [C] float32 = final |grad f_c| / |grad f_c(0)| (b, iters, gnorm may be
 * NULL).  workspace: se_linear_svm_workspace_bytes(N, D, C) bytes of device memory, 256-byte aligned.
 * The call BLOCKS: the host reads the classes' convergence flags after every CG step, so it synchronises with `stream`
 * and cannot be captured into a CUDA graph (SE_ERR_ARG inside a capture). */
int64_t se_linear_svm_workspace_bytes(int N, int D, int C);
int se_linear_svm_fit(const float* X, int64_t ldx, int N, int D, const int32_t* labels, int C, float penalty, float tol,
                      int max_iter, float* W, float* b, int32_t* iters, float* gnorm, void* workspace, void* stream);
/* Feature scaling of train_and_predict (:33-38) with numpy's float32 results bit for bit, and score negation:
 *   SE_SCALE_ROW_L2      y = x / ||x||_2 per row (float32 squares summed in numpy's pairwise order, true division)
 *   SE_SCALE_COL_MAXABS  colmax[j] = max_i |x_ij|          (y is not written)
 *   SE_SCALE_COL_DIV     y = x / max(1e-8, colmax[j])      (true division)
 *   SE_SCALE_MUL         y = scale * x                     (scale = -1 turns se_row_topk's ascending order descending)
 * x [rows, ldx], y [rows, ldy]; y may be x. */
#define SE_SCALE_ROW_L2 0
#define SE_SCALE_COL_MAXABS 1
#define SE_SCALE_COL_DIV 2
#define SE_SCALE_MUL 3
int se_scale_features(const float* x, int64_t ldx, int rows, int D, int op, float* colmax, float scale, float* y, int64_t ldy,
                      void* stream);

/* ------------------------------------------------------------------ class embeddings (compute_class_embedding.py)
 * float64 throughout (csrc/class_embed.cu).  D [C, ldd] is the LCS-height distance table, S = 1 - D. */
#define SE_ERR_NOT_CONVERGED (-4)
/* D_ij = heights[first common entry of the lists of i and j] / max_height, D_ii = 0.  Class c's list is
 * ancestors[offsets[c] .. offsets[c+1]), its ancestors and itself as node ranks in the order (-depth, node index),
 * ascending; heights is indexed by rank.  max_len = the longest list (SE_ERR_UNSUPPORTED above 64).  A pair without a
 * common ancestor gets NaN. */
int se_lcs_height_table(const int32_t* offsets, const int32_t* ancestors, const int32_t* heights, int max_height, int C,
                        int max_len, double* D, int64_t ldd, void* stream);
/* In place: A [n, lda] symmetric (its lower triangle is read) -> its lower Cholesky factor L, upper triangle zeroed.
 * status (device int): -1, or the first row whose pivot is <= 0 or NaN; that row's diagonal then holds the pivot and
 * the rows after it are meaningless. */
int se_cholesky_f64(double* A, int64_t lda, int n, int32_t* status, void* stream);
/* SE_GRAM_SIM: out [C, C] = 1 - D.  SE_GRAM_SPHERES: out [C-1, C-1] = (D_0,i+1^2 + D_0,j+1^2 - D_i+1,j+1^2) / 2, the Gram
 * matrix of the classes placed relative to class 0. */
#define SE_GRAM_SIM 0
#define SE_GRAM_SPHERES 1
int se_class_gram_f64(const double* D, int64_t ldd, int C, int op, double* out, int64_t ldo, void* stream);
/* X [m, ldx]: SE_COL_SQNORM out[j] = sum_i X_ij^2;  SE_COL_CENTER X_ij -= mean_i X_ij (out unused). */
#define SE_COL_SQNORM 0
#define SE_COL_CENTER 1
int se_column_op_f64(double* X, int64_t ldx, int m, int n, int op, double* out, void* stream);
/* Y[:, c] = X[:, cols[c]] for c < k (cols on the device) */
int se_gather_columns_f64(const double* X, int64_t ldx, int m, const int32_t* cols, int k, double* Y, int64_t ldy, void* stream);
/* X_i /= ||X_i||_2 for every row */
int se_row_normalize_f64(double* X, int64_t ldx, int m, int n, void* stream);
/* One-sided block Jacobi, in place: right-multiplies X [m, ldx] by plane rotations until every pair of its n columns
 * satisfies |a.b| <= n eps |a| |b| (pairs with a zero column excepted) over a whole sweep.  Blocks of 16 columns meet in
 * a fixed round-robin order, so reruns give the same bits.  *sweeps (host) = the sweeps run, the last one included;
 * SE_ERR_NOT_CONVERGED after max_sweeps.  workspace: se_jacobi_columns_workspace_bytes(m, n) bytes of device memory.
 * The call BLOCKS (it reads the convergence flag after every sweep) and cannot be captured into a CUDA graph. */
int64_t se_jacobi_columns_workspace_bytes(int m, int n);
int se_jacobi_columns_f64(double* X, int64_t ldx, int m, int n, int max_sweeps, int32_t* sweeps, void* workspace, void* stream);
/* The self-check of compute_class_embedding.py over all C^2 pairs (diagonal included): out (device) [2] = max and mean of
 * SE_DEV_SIM |E_i.E_j - (1 - D_ij)| or SE_DEV_DIST | ||E_i - E_j|| - D_ij |, E [C, lde] with dim columns.  Tiles are
 * combined in a fixed order.  workspace: se_embedding_deviation_workspace_bytes(C) bytes of device memory. */
#define SE_DEV_SIM 0
#define SE_DEV_DIST 1
int64_t se_embedding_deviation_workspace_bytes(int C);
int se_embedding_deviation_f64(const double* E, int64_t lde, int C, int dim, const double* D, int64_t ldd, int mode, double* out,
                               void* workspace, void* stream);

/* ------------------------------------------------------------------ plan runner
 * Runs a host-built array of ops (one training step is ~900 launches) in one call so that
 * neither Python nor ctypes sits between launches.  Each op is an opcode plus the argument
 * block of the entry point above it maps to (see semantic_embeddings_b200/engine.py). */
typedef struct {
  int32_t opcode;
  int32_t i[15];
  float f[8];
  void* p[16];
} se_op;
int se_run_ops(const se_op* ops, int n, int mode, void* stream);
/* profiling variant (bench.py): eager, a CUDA-event pair around every op, per-op device milliseconds */
int se_run_ops_timed(const se_op* ops, int n, int mode, void* stream, float* ms_out);

#ifdef __cplusplus
}
#endif
#endif /* SE_B200_H */
