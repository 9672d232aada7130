// C-ABI glue: error state, launch counter, conv/dense dispatch between the arithmetic modes,
// and the plan runner (se_run_ops) that issues a whole training step without returning to Python.
#include <stdarg.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>

#include "common.cuh"
#include "conv_plan.cuh"
#include "opcodes.h"

namespace se {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};
static int g_sms = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
bool pdl_enabled() {
  static const bool on = getenv("SE_NO_PDL") == nullptr;
  return on;
}
bool coop_enabled() {
  static const bool on = getenv("SE_BN_COOP") != nullptr;
  return on;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
int sm_count() {
  if (g_sms == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess &&
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      g_sms = n;
    else
      g_sms = 148;
  }
  return g_sms;
}

// conv_simt.cu
int conv_fwd_simt(const se_conv_desc*, const float*, const float*, const float*, const float*, float*, int, double*, cudaStream_t);
int conv_dgrad_simt(const se_conv_desc*, const float*, const float*, float*, float, cudaStream_t);
int conv_wgrad_simt(const se_conv_desc*, const float*, const float*, float*, float*, cudaStream_t);

static int check_desc(const se_conv_desc* d) {
  if (!d) { set_error("null conv descriptor"); return SE_ERR_ARG; }
  if (d->N <= 0 || d->H <= 0 || d->W <= 0 || d->Cin <= 0 || d->Cout <= 0 || d->kh <= 0 || d->kw <= 0 ||
      d->stride <= 0 || d->Ho <= 0 || d->Wo <= 0 || d->pad_t < 0 || d->pad_l < 0) {
    set_error("invalid conv descriptor");
    return SE_ERR_ARG;
  }
  // the last window must start inside the (top/left padded) input
  if ((d->Ho - 1) * d->stride - d->pad_t >= d->H || (d->Wo - 1) * d->stride - d->pad_l >= d->W) {
    set_error("conv output size inconsistent with input/stride/padding");
    return SE_ERR_ARG;
  }
  return SE_OK;
}

}  // namespace se

using namespace se;

extern "C" const char* se_version(void) { return "se_b200 0.1 (sm_90a)"; }
extern "C" const char* se_last_error(void) { return g_err; }
extern "C" int64_t se_launch_count(void) { return g_launches.load(); }
extern "C" int se_device_sm_count(void) { return sm_count(); }
namespace se { int init_conv_simt(); int init_pairwise_tc(); int init_conv_tc(); int init_conv_wgrad_tc(); int init_head(); }
// One-time per-process setup that must not happen inside a CUDA-graph capture: device query and the
// cudaFuncSetAttribute calls of every kernel that needs more than 48 KB of dynamic shared memory.
static bool side_stream_ready();
static int prepare_side_workspace();

extern "C" int se_init(void) {
  sm_count();
  int rc = se::init_conv_simt();
  if (rc == SE_OK) rc = se::init_pairwise_tc();
  if (rc == SE_OK) rc = se::init_conv_tc();
  if (rc == SE_OK) rc = se::init_conv_wgrad_tc();
  if (rc == SE_OK) rc = se::init_head();
  if (rc == SE_OK) side_stream_ready();      // side stream + fork/join events of se_run_ops exist before any graph capture
  if (rc == SE_OK) rc = prepare_side_workspace();   // and the weight-gradient workspace of that stream
  return rc;
}
namespace se { int tc_capabilities(); }
extern "C" int se_tc_capabilities(void) { return se::tc_capabilities(); }

extern "C" int se_conv2d_fwd_aux(const se_conv_desc* d, const float* x, const float* w, const se_conv_aux* aux,
                                 const float* bias, const float* residual, float* y, int relu, double* stats, int mode,
                                 void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(x && w && y, "null pointer");
  ConvCall c;
  c.w_t = aux && aux->w_t;
  c.w_t_lo = aux && aux->w_t_lo;
  c.stats = stats != nullptr;
  ConvPlan pl;
  if (conv_plan(d, 0, mode, c, &pl) == CONV_FP32) return conv_fwd_simt(d, x, w, bias, residual, y, relu, stats, as_stream(stream));
  rc = conv_fwd_tc(pl, d, x, aux->w_t, aux->w_t_lo, bias, residual, y, relu, pl.fused_stats ? stats : nullptr, as_stream(stream));
  if (rc || !stats || pl.fused_stats) return rc;
  return se_bn_stats(y, (int64_t)d->N * d->Ho * d->Wo, d->Cout, stats, stream);
}

extern "C" int se_conv2d_fwd_ex(const se_conv_desc* d, const float* x, const float* w, const float* w_t,
                                const float* bias, const float* residual, float* y, int relu, double* stats, int mode,
                                void* stream) {
  se_conv_aux aux = {w_t, nullptr, nullptr};
  return se_conv2d_fwd_aux(d, x, w, &aux, bias, residual, y, relu, stats, mode, stream);
}

extern "C" int se_conv_bn_fwd(const se_conv_desc* d, const float* x, const float* w, const float* w_t, const float* bias,
                              float* y, int relu, double* stats, const float* gamma, const float* beta, float eps,
                              float momentum, float* moving_mean, float* moving_var, float* save_mean, float* save_invstd,
                              const float* res, int bn_relu, float* bn_out, void* counter, int mode, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(x && w && y && stats && gamma && beta && save_mean && save_invstd && bn_out, "null pointer");
  (void)counter;
  rc = se_conv2d_fwd_ex(d, x, w, w_t, bias, nullptr, y, relu, stats, mode, stream);
  if (rc) return rc;
  se_residual r;
  r.ptr = res; r.C = d->Cout; r.pad_lo = 0; r.pool = 1; r.H = d->Ho; r.W = d->Wo;
  return se_bn_fwd_train(y, (int64_t)d->N * d->Ho * d->Wo, d->Cout, stats, gamma, beta, eps, momentum, moving_mean, moving_var,
                         save_mean, save_invstd, res ? &r : nullptr, bn_relu, bn_out, stream);
}

extern "C" int se_conv2d_fwd(const se_conv_desc* d, const float* x, const float* w, const float* bias,
                             const float* residual, float* y, int relu, double* stats, int mode, void* stream) {
  return se_conv2d_fwd_ex(d, x, w, nullptr, bias, residual, y, relu, stats, mode, stream);
}

namespace se {
int transpose_filters(const float* P, float* PT, float* PL, float* PTL, const long long* table, int n, cudaStream_t st);
}
extern "C" int se_transpose_filters(const float* P, float* PT, const int64_t* table, int n, void* stream) {
  SE_REQUIRE(P && PT && table && n >= 0, "bad arguments");
  return se::transpose_filters(P, PT, nullptr, nullptr, reinterpret_cast<const long long*>(table), n, as_stream(stream));
}
extern "C" int se_split_filters(const float* P, float* PT, float* PL, float* PTL, const int64_t* table, int n, void* stream) {
  SE_REQUIRE(P && PT && PL && PTL && table && n >= 0, "bad arguments");
  return se::transpose_filters(P, PT, PL, PTL, reinterpret_cast<const long long*>(table), n, as_stream(stream));
}

extern "C" int se_conv2d_dgrad_aux(const se_conv_desc* d, const float* dy, const float* w, const se_conv_aux* aux, float* dx,
                                   float beta, int mode, void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(dy && w && dx, "null pointer");
  ConvCall c;
  c.w_lo = aux && aux->w_lo;
  c.beta = beta;
  ConvPlan pl;
  if (conv_plan(d, 1, mode, c, &pl) == CONV_FP32) return conv_dgrad_simt(d, dy, w, dx, beta, as_stream(stream));
  return conv_dgrad_tc(pl, d, dy, w, c.w_lo ? aux->w_lo : nullptr, dx, beta, as_stream(stream));
}
extern "C" int se_conv2d_dgrad(const se_conv_desc* d, const float* dy, const float* w, float* dx, float beta, int mode,
                               void* stream) {
  return se_conv2d_dgrad_aux(d, dy, w, nullptr, dx, beta, mode, stream);
}

extern "C" int se_conv2d_path(const se_conv_desc* d, int mode, int direction) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(direction >= 0 && direction <= 2, "direction: 0 forward, 1 backward data, 2 weight gradient");
  ConvPlan pl;
  return conv_plan(d, direction, mode, ConvCall(), &pl) == CONV_FP32 ? 0 : 1;
}

extern "C" int se_conv2d_wgrad(const se_conv_desc* d, const float* x, const float* dy, float* dw, float* dbias, int mode,
                               void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(x && dy && dw, "null pointer");
  // the kernel stores dW / dbias as float2 / float4
  ConvCall c;
  c.aligned = (reinterpret_cast<uintptr_t>(dw) & 15) == 0 && (reinterpret_cast<uintptr_t>(dbias) & 15) == 0;
  c.sms = sm_count();
  ConvPlan pl;
  if (conv_plan(d, 2, mode, c, &pl) == CONV_FP32) return conv_wgrad_simt(d, x, dy, dw, dbias, as_stream(stream));
  return conv_wgrad_tc(pl, x, dy, dw, dbias, as_stream(stream));
}

static se_conv_desc dense_desc(int B, int Cin, int Cout) {
  se_conv_desc d;
  d.N = B; d.H = 1; d.W = 1; d.Cin = Cin; d.Cout = Cout; d.kh = 1; d.kw = 1; d.stride = 1; d.pad_t = 0; d.pad_l = 0;
  d.Ho = 1; d.Wo = 1;
  return d;
}

extern "C" int se_dense_fwd(const float* x, const float* w, const float* bias, float* y, int B, int Cin, int Cout,
                            int relu, double* stats, int mode, void* stream) {
  se_conv_desc d = dense_desc(B, Cin, Cout);
  return se_conv2d_fwd(&d, x, w, bias, nullptr, y, relu, stats, mode, stream);
}

extern "C" int se_dense_bwd(const float* x, const float* w, const float* dy, float* dx, float beta, float* dw,
                            float* dbias, int B, int Cin, int Cout, int mode, void* stream) {
  se_conv_desc d = dense_desc(B, Cin, Cout);
  int rc = SE_OK;
  if (dx) rc = se_conv2d_dgrad(&d, dy, w, dx, beta, mode, stream);
  if (rc) return rc;
  if (dw) rc = se_conv2d_wgrad(&d, x, dy, dw, dbias, mode, stream);
  return rc;
}

// ---------------------------------------------------------------------------------------- plan runner
static se_conv_desc desc_from(const int32_t* i) {
  se_conv_desc d;
  d.N = i[0]; d.H = i[1]; d.W = i[2]; d.Cin = i[3]; d.Cout = i[4]; d.kh = i[5]; d.kw = i[6]; d.stride = i[7];
  d.pad_t = i[8]; d.pad_l = i[9]; d.Ho = i[10]; d.Wo = i[11];
  return d;
}

extern "C" int se_sgd_apply_devlr(float* p, const float* g, float* v, int64_t n, const float* lr_dev, float momentum,
                                  int nesterov, float clipnorm, const double* out, void* stream);

// Weight gradients are off the critical path of the backward pass (nothing reads dW before the optimizer), so a
// multi-op plan issues them on a second, lowest-priority stream: fork after the op that produced dY, join at the end of
// the plan.  Inside a CUDA-graph capture this becomes a parallel branch.  The backward-data / BatchNorm-backward
// chain and the wgrad kernels can share an SM (shared memory, registers; see
// conv_tc.cu / conv_wgrad_tc.cu), so the side branch fills the latency bubbles of the main chain.  SE_NO_SIDE_STREAM=1
// keeps everything on one stream.
static cudaStream_t g_side = nullptr;
static cudaEvent_t g_ev_fork = nullptr, g_ev_join = nullptr;
static bool side_stream_ready() {
  static const bool off = getenv("SE_NO_SIDE_STREAM") != nullptr;
  if (off) return false;
  if (!g_side) {
    int lo = 0, hi = 0;
    if (cudaDeviceGetStreamPriorityRange(&lo, &hi) != cudaSuccess) return false;
    if (cudaStreamCreateWithPriority(&g_side, cudaStreamNonBlocking, lo) != cudaSuccess) { g_side = nullptr; return false; }
    if (cudaEventCreateWithFlags(&g_ev_fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_join, cudaEventDisableTiming) != cudaSuccess) {
      g_side = nullptr;
      return false;
    }
  }
  return true;
}

namespace se { int wgrad_workspace_prepare(cudaStream_t st); }
static int prepare_side_workspace() { return g_side ? se::wgrad_workspace_prepare(g_side) : SE_OK; }

namespace se {
cudaStream_t comm_stream();
bool comm_ready();
int comm_allreduce_ranges(float* base, const long long* off, const long long* cnt, int nranges, cudaStream_t st);
}
static cudaEvent_t g_ev_comm_main = nullptr, g_ev_comm_side = nullptr, g_ev_comm_done = nullptr;
static bool g_comm_pending = false;      // all-reduces in flight on the communication stream (joined before the optimizer)
static bool comm_events_ready() {
  if (!g_ev_comm_main) {
    if (cudaEventCreateWithFlags(&g_ev_comm_main, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_comm_side, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&g_ev_comm_done, cudaEventDisableTiming) != cudaSuccess) {
      g_ev_comm_main = nullptr;
      return false;
    }
  }
  return true;
}
static void join_comm(void* stream) {
  if (g_comm_pending) {
    cudaEventRecord(g_ev_comm_done, se::comm_stream());
    cudaStreamWaitEvent(as_stream(stream), g_ev_comm_done, 0);
    g_comm_pending = false;
  }
}

static int run_ops_impl(const se_op* ops, int n, int mode, void* stream, bool* forked);

extern "C" int se_run_ops(const se_op* ops, int n, int mode, void* stream) {
  SE_REQUIRE(ops && n >= 0, "bad arguments");
  bool forked = false;
  int rc = run_ops_impl(ops, n, mode, stream, &forked);
  if (forked) {   // join on every path (an unjoined fork would invalidate an ongoing capture)
    cudaEventRecord(g_ev_join, g_side);
    cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
  }
  join_comm(stream);
  return rc;
}

static int run_ops_impl(const se_op* ops, int n, int mode, void* stream, bool* forked) {
  const bool use_side = n > 1 && side_stream_ready();
  bool transposing = false;          // filter transposition in flight on the side stream
  for (int k = 0; k < n; ++k) {
    const se_op& o = ops[k];
    const int32_t* i = o.i;
    const float* f = o.f;
    void* const* p = o.p;
    int rc = SE_OK;
    switch (o.opcode) {
      case SE_OP_CONV_FWD: {
        se_conv_desc d = desc_from(i);
        if (transposing && p[6]) {   // first consumer of the transposed filters: the side branch joins here
          cudaEventRecord(g_ev_join, g_side);
          cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
          transposing = false;
          *forked = false;
        }
        se_conv_aux aux = {(const float*)p[6], (const float*)p[7], nullptr};
        rc = se_conv2d_fwd_aux(&d, (const float*)p[0], (const float*)p[1], &aux, (const float*)p[2],
                               (const float*)p[3], (float*)p[4], i[12], (double*)p[5], i[13] >= 0 ? i[13] : mode, stream);
        break;
      }
      case SE_OP_CONV_BN_FWD: {
        // p: 0 x, 1 w, 2 bias, 3 y, 4 stats, 5 w_t, 6 gamma, 7 beta, 8 moving_mean, 9 moving_var, 10 save_mean,
        //    11 save_invstd, 12 residual, 13 bn_out, 14 counter;  i[12] conv relu, i[14] bn relu;  f: eps, momentum
        se_conv_desc d = desc_from(i);
        if (transposing && p[5]) {
          cudaEventRecord(g_ev_join, g_side);
          cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
          transposing = false;
          *forked = false;
        }
        rc = se_conv_bn_fwd(&d, (const float*)p[0], (const float*)p[1], (const float*)p[5], (const float*)p[2], (float*)p[3],
                            i[12], (double*)p[4], (const float*)p[6], (const float*)p[7], f[0], f[1], (float*)p[8],
                            (float*)p[9], (float*)p[10], (float*)p[11], (const float*)p[12], i[14], (float*)p[13], p[14],
                            i[13] >= 0 ? i[13] : mode, stream);
        break;
      }
      case SE_OP_CONV_DGRAD: {
        se_conv_desc d = desc_from(i);
        se_conv_aux aux = {nullptr, nullptr, (const float*)p[3]};
        rc = se_conv2d_dgrad_aux(&d, (const float*)p[0], (const float*)p[1], &aux, (float*)p[2], f[0],
                                 i[13] >= 0 ? i[13] : mode, stream);
        break;
      }
      case SE_OP_CONV_WGRAD: {
        se_conv_desc d = desc_from(i);
        void* ws = stream;
        if (use_side) {
          cudaEventRecord(g_ev_fork, as_stream(stream));
          cudaStreamWaitEvent(g_side, g_ev_fork, 0);
          ws = g_side;
          *forked = true;
        }
        rc = se_conv2d_wgrad(&d, (const float*)p[0], (const float*)p[1], (float*)p[2], (float*)p[3], i[13] >= 0 ? i[13] : mode, ws);
        break;
      }
      case SE_OP_BN_STATS:
        rc = se_bn_stats((const float*)p[0], i[1], i[0], (double*)p[1], stream);
        break;
      case SE_OP_BN_FWD_TRAIN:
      case SE_OP_BN_FWD_INFER: {
        se_residual r;
        r.ptr = (const float*)p[8]; r.C = i[3]; r.pad_lo = i[4]; r.pool = i[5]; r.H = i[6]; r.W = i[7];
        if (o.opcode == SE_OP_BN_FWD_TRAIN)
          rc = se_bn_fwd_train((const float*)p[0], i[1], i[0], (const double*)p[1], (const float*)p[2], (const float*)p[3],
                               f[0], f[1], (float*)p[4], (float*)p[5], (float*)p[6], (float*)p[7], &r, i[2], (float*)p[9], stream);
        else
          rc = se_bn_fwd_infer((const float*)p[0], i[1], i[0], (const float*)p[2], (const float*)p[3], (const float*)p[4],
                               (const float*)p[5], f[0], &r, i[2], (float*)p[9], stream);
        break;
      }
      case SE_OP_BN_BWD:
        rc = se::bn_bwd((const float*)p[0], (const float*)p[1], (const float*)p[2], i[1], i[0], (const float*)p[3],
                        (const float*)p[4], (const float*)p[5], i[2], i[3], (float*)p[6], f[0], (float*)p[7], f[1],
                        (float*)p[8], (float*)p[9], (double*)p[10], i[4], stream);
        break;
      case SE_OP_SHORTCUT_BWD: {
        se_residual r;
        r.ptr = (const float*)p[2]; r.C = i[5]; r.pad_lo = i[6]; r.pool = i[7]; r.H = i[1]; r.W = i[2];
        rc = se_shortcut_bwd((const float*)p[0], (const float*)p[1], i[4], i[0], i[1], i[2], i[3], &r, (float*)p[2], f[0], stream);
        break;
      }
      case SE_OP_AVGPOOL_FWD:
        rc = se_avgpool2_fwd((const float*)p[0], (float*)p[1], i[0], i[1], i[2], i[3], stream);
        break;
      case SE_OP_AVGPOOL_BWD:
        rc = se_avgpool2_bwd((const float*)p[0], (float*)p[1], f[0], i[0], i[1], i[2], i[3], stream);
        break;
      case SE_OP_MAXPOOL_FWD:
        rc = se_maxpool_fwd((const float*)p[0], (float*)p[1], i[0], i[1], i[2], i[3], i[4], i[5], i[6], i[7], i[8], i[9], stream);
        break;
      case SE_OP_MAXPOOL_BWD:
        rc = se_maxpool_bwd((const float*)p[0], (const float*)p[1], (const float*)p[2], (float*)p[3], i[0], i[1], i[2],
                            i[3], i[4], i[5], i[6], i[7], i[8], i[9], stream);
        break;
      case SE_OP_GAP_FWD:
        rc = se_gap_fwd((const float*)p[0], (float*)p[1], i[0], i[1], i[2], stream);
        break;
      case SE_OP_GAP_BWD:
        rc = se_gap_bwd((const float*)p[0], (float*)p[1], f[0], i[0], i[1], i[2], stream);
        break;
      case SE_OP_ADD_FWD:
        rc = se_add_fwd((const float*)p[0], (const float*)p[1], (float*)p[2], i[1], i[0], stream);
        break;
      case SE_OP_ADD_BWD:
        rc = se_add_bwd((const float*)p[0], (const float*)p[1], i[0], (float*)p[2], f[0], (float*)p[3], f[1], i[1], stream);
        break;
      case SE_OP_HEAD:
        // i[5] = SE_LOSS_DEVISE_RANK: the ranking loss with the margin in f[1] (0 in every other head op)
        if (i[5] == SE_LOSS_DEVISE_RANK)
          rc = se_devise_rank_fwd_bwd((const float*)p[0], i[0], (const int32_t*)p[1], (const float*)p[2], i[1], i[2], i[3],
                                      i[4], i[5], f[0], (const float*)p[3], (float*)p[4], (float*)p[5], (float*)p[6],
                                      (float*)p[7], (float*)p[8], f[1], stream);
        else
          rc = se_embed_head_fwd_bwd_ex((const float*)p[0], i[0], (const int32_t*)p[1], (const float*)p[2], i[1], i[2], i[3],
                                      i[4], i[5], f[0], (const float*)p[3], (float*)p[4], (float*)p[5], (float*)p[6],
                                      (float*)p[7], (float*)p[8], stream);
        break;
      case SE_OP_XENT:
        // f[1] = label smoothing (learn_classifier.py --label_smoothing); 0 in every embedding-training plan
        if (f[1] != 0.f)
          rc = se_softmax_xent_smooth_fwd_bwd((const float*)p[0], i[0], (const int32_t*)p[1], i[1], i[2], f[1], f[0],
                                              (float*)p[2], (float*)p[3], (float*)p[4], (float*)p[5], (float*)p[6], stream);
        else
          rc = se_softmax_xent_fwd_bwd_ex((const float*)p[0], i[0], (const int32_t*)p[1], i[1], i[2], f[0], (float*)p[2],
                                          (float*)p[3], (float*)p[4], (float*)p[5], (float*)p[6], stream);
        break;
      case SE_OP_LABELEMBED:
        // i: ld, ldE, B, C;  f: scale, tau, alpha, beta;
        // p: 0 out1, 1 out2, 2 labels, 3 table, 4 loss, 5 acc, 6 d_out1, 7 d_out2, 8 d_table, 9 workspace
        rc = se_labelembed_fwd_bwd((const float*)p[0], (const float*)p[1], i[0], (const int32_t*)p[2], (const float*)p[3],
                                   i[1], i[2], i[3], f[1], f[2], f[3], f[0], (float*)p[4], (float*)p[5], (float*)p[6],
                                   (float*)p[7], (float*)p[8], p[9], stream);
        break;
      case SE_OP_CENTER_LOSS:
        // i: ldz, ldc, B, C, D;  f: scale (the loss weight over the global batch);
        // p: 0 z, 1 labels, 2 centroids, 3 loss, 4 d_z, 5 d_centroids
        rc = se_center_loss_fwd_bwd((const float*)p[0], i[0], (const int32_t*)p[1], (const float*)p[2], i[1], i[2], i[3],
                                    i[4], f[0], (float*)p[3], (float*)p[4], (float*)p[5], stream);
        break;
      case SE_OP_MEMSET: {
        if (i[0] & 1) {
          // a memset of GRADIENT memory (frozen parameters, Engine.set_trainable): the weight-gradient kernels of the side
          // stream and the all-reduces of the communication stream write that memory -- join them first
          join_comm(stream);
          if (*forked) {
            cudaEventRecord(g_ev_join, g_side);
            cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
            *forked = false;
          }
        }
        cudaError_t e = cudaMemsetAsync(p[0], 0, (size_t)(uintptr_t)p[1], as_stream(stream));
        if (e != cudaSuccess) { set_error("memset: %s", cudaGetErrorString(e)); rc = SE_ERR_CUDA; }
        break;
      }
      case SE_OP_TRANSPOSE_FILTERS:
        if (mode == SE_MODE_TF32 || mode == SE_MODE_TF32X3) {
          // the transposed filter copies are first needed by the first tensor-core convolution: the transposition runs
          // on the side stream beside the statistics memset, the stem convolution and its BatchNorm
          void* ts = stream;
          if (use_side && !*forked) {
            cudaEventRecord(g_ev_fork, as_stream(stream));
            cudaStreamWaitEvent(g_side, g_ev_fork, 0);
            ts = g_side;
            *forked = true;
            transposing = true;
          }
          if (mode == SE_MODE_TF32X3 && p[3] && p[4])
            rc = se_split_filters((const float*)p[0], (float*)p[1], (float*)p[3], (float*)p[4], (const int64_t*)p[2], i[0], ts);
          else
            rc = se_transpose_filters((const float*)p[0], (float*)p[1], (const int64_t*)p[2], i[0], ts);
        }
        break;
      case SE_OP_ALLREDUCE: {
        // p[0] = flat gradient buffer, i[0] = number of ranges, p[1 + 2k] / p[2 + 2k] = element offset / count of range k.
        // The ranges hold gradients that every op up to here has finished writing: weight gradients on the side stream,
        // BatchNorm / bias gradients on the main stream.  The exchange runs on the communication stream behind both and
        // overlaps the rest of the backward pass; the optimizer joins it.
        if (!se::comm_ready() || !comm_events_ready()) { set_error("SE_OP_ALLREDUCE without a communicator (se_comm_init)"); return SE_ERR_ARG; }
        cudaStream_t cs = se::comm_stream();
        cudaEventRecord(g_ev_comm_main, as_stream(stream));
        cudaStreamWaitEvent(cs, g_ev_comm_main, 0);
        if (*forked) {
          cudaEventRecord(g_ev_comm_side, g_side);
          cudaStreamWaitEvent(cs, g_ev_comm_side, 0);
        }
        long long off[7], cnt[7];
        const int nr = i[0] < 7 ? i[0] : 7;
        for (int r = 0; r < nr; ++r) { off[r] = (long long)(uintptr_t)p[1 + 2 * r]; cnt[r] = (long long)(uintptr_t)p[2 + 2 * r]; }
        rc = se::comm_allreduce_ranges((float*)p[0], off, cnt, nr, cs);
        g_comm_pending = true;
        break;
      }
      case SE_OP_SGD_PREPARE:
        join_comm(stream);
        if (*forked) {   // the optimizer reads every gradient: the side branch joins here
          cudaEventRecord(g_ev_join, g_side);
          cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
          *forked = false;
        }
        rc = se_sgd_prepare((const float*)p[0], (float*)p[1], (int64_t)(uintptr_t)p[2], (const se_l2_segment*)p[3], i[0],
                            (double*)p[4], stream);
        break;
      case SE_OP_SGD_APPLY:
        if (*forked) {
          cudaEventRecord(g_ev_join, g_side);
          cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
          *forked = false;
        }
        // p[3] = lr_state {lr, decay, iterations, lr_t}: the schedule kernel derives this step's lr_t, the update reads it
        rc = se_sgd_schedule((float*)p[3], stream);
        if (rc == SE_OK)
          rc = se_sgd_apply_devlr((float*)p[0], (const float*)p[1], (float*)p[5], (int64_t)(uintptr_t)p[2],
                                  (const float*)p[3] + 3, f[0], i[0], f[1], (const double*)p[4], stream);
        break;
      case SE_OP_ADAGRAD_APPLY:
        // the Adagrad update in place of SGD_APPLY: same p[0..5] (p[5] = accumulators), f[0] = epsilon, f[1] = clipnorm
        if (*forked) {
          cudaEventRecord(g_ev_join, g_side);
          cudaStreamWaitEvent(as_stream(stream), g_ev_join, 0);
          *forked = false;
        }
        rc = se_sgd_schedule((float*)p[3], stream);
        if (rc == SE_OK)
          rc = se_adagrad_apply_devlr((float*)p[0], (const float*)p[1], (float*)p[5], (int64_t)(uintptr_t)p[2],
                                      (const float*)p[3] + 3, f[0], f[1], (const double*)p[4], stream);
        break;
      default:
        set_error("se_run_ops: unknown opcode %d at index %d", o.opcode, k);
        return SE_ERR_ARG;
    }
    if (rc != SE_OK) return rc;
  }
  return SE_OK;
}


// Profiling variant used by bench.py: runs the ops eagerly with a CUDA-event pair around each one and
// returns the per-op device time in milliseconds (ms_out[n]).  Not capturable.
extern "C" int se_run_ops_timed(const se_op* ops, int n, int mode, void* stream, float* ms_out) {
  SE_REQUIRE(ops && ms_out && n >= 0, "bad arguments");
  cudaStream_t st = as_stream(stream);
  cudaEvent_t* ev = new cudaEvent_t[2 * (size_t)n];
  for (int k = 0; k < 2 * n; ++k) cudaEventCreate(&ev[k]);
  int rc = SE_OK;
  for (int k = 0; k < n && rc == SE_OK; ++k) {
    cudaEventRecord(ev[2 * k], st);
    rc = se_run_ops(ops + k, 1, mode, stream);
    cudaEventRecord(ev[2 * k + 1], st);
  }
  cudaStreamSynchronize(st);
  for (int k = 0; k < n; ++k) {
    ms_out[k] = 0.f;
    if (rc == SE_OK) cudaEventElapsedTime(&ms_out[k], ev[2 * k], ev[2 * k + 1]);
  }
  for (int k = 0; k < 2 * n; ++k) cudaEventDestroy(ev[k]);
  delete[] ev;
  return rc;
}
