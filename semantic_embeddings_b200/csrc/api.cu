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
// set while se_run_ops_runner issues a plan: its grid-barrier kernels are launched cooperatively (see there)
static thread_local bool t_runner_plan = false;
bool coop_enabled() {
  static const bool on = getenv("SE_BN_COOP") != nullptr;
  return on || t_runner_plan;
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
// Weight gradients are off the critical path of the backward pass (nothing reads dW before the optimizer), so a
// multi-op plan issues them on a second, lowest-priority stream (see Streams below).  Inside a CUDA-graph capture this
// becomes a parallel branch.  The backward-data / BatchNorm-backward chain and the wgrad kernels can share an SM (shared
// memory, registers; see conv_tc.cu / conv_wgrad_tc.cu), so the side branch fills the latency bubbles of the main chain.
// A plan runner owns that side stream, its fork / join events and, through the side stream, a weight-gradient workspace
// (wgrad_workspace is keyed by stream).  se_run_ops runs on the default runner that se_init creates; se_runner_create
// makes one more for every plan that runs at the same time as another (see se_run_ops_runner).
struct se_runner {
  cudaStream_t side = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
};
static se_runner g_default_runner;

namespace se {
int init_conv_simt(); int init_pairwise_tc(); int init_conv_tc(); int init_conv_wgrad_tc(); int init_head();
int init_bn_bwd(); int init_row_topk(); int init_resample_crop();
int wgrad_workspace_prepare(cudaStream_t st);
void wgrad_workspace_release(cudaStream_t st);

static void runner_free(se_runner* r) {
  if (r->side) {
    cudaStreamSynchronize(r->side);
    wgrad_workspace_release(r->side);
    cudaStreamDestroy(r->side);
  }
  if (r->ev_fork) cudaEventDestroy(r->ev_fork);
  if (r->ev_join) cudaEventDestroy(r->ev_join);
  *r = se_runner();
}

// the side stream (lowest priority), its events and its weight-gradient workspace: all allocated here, never inside a
// capture
static int runner_init(se_runner* r) {
  int lo = 0, hi = 0;
  cudaError_t e = cudaDeviceGetStreamPriorityRange(&lo, &hi);
  if (e == cudaSuccess) e = cudaStreamCreateWithPriority(&r->side, cudaStreamNonBlocking, lo);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r->ev_fork, cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreateWithFlags(&r->ev_join, cudaEventDisableTiming);
  if (e != cudaSuccess) {
    set_error("cannot create the side stream of a plan runner: %s", cudaGetErrorString(e));
    runner_free(r);
    return SE_ERR_CUDA;
  }
  const int rc = wgrad_workspace_prepare(r->side);
  if (rc) runner_free(r);
  return rc;
}

static int setup() {
  sm_count();
  for (int (*init)() : {init_conv_simt, init_pairwise_tc, init_conv_tc, init_conv_wgrad_tc, init_head, init_bn_bwd,
                        init_row_topk, init_resample_crop}) {
    const int rc = init();
    if (rc) return rc;
  }
  return runner_init(&g_default_runner);
}

int ensure_setup() {
  static char msg[sizeof(g_err)];
  static const int rc = [] {
    const int r = setup();
    if (r) snprintf(msg, sizeof(msg), "%s", g_err);
    return r;
  }();
  if (rc) set_error("%s", msg);
  return rc;
}
}  // namespace se

extern "C" int se_init(void) { return ensure_setup(); }
namespace se { int tc_capabilities(); }
extern "C" int se_tc_capabilities(void) { return se::tc_capabilities(); }

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" int se_conv2d_fwd_aux(const se_conv_desc* d, const float* x, const float* w, const se_conv_aux* aux,
                                 const float* bias, const float* residual, float* y, int relu, double* stats, int mode,
                                 void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(x && w && y, "null pointer");
  if ((rc = ensure_setup())) return rc;
  ConvCall c;
  c.w_t = aux && aux->w_t;
  c.w_t_lo = aux && aux->w_t_lo;
  c.stats = stats != nullptr;
  c.x_aligned = aligned16(x);
  c.y_aligned = aligned16(y);
  c.residual = residual != nullptr;
  c.sms = sm_count();
  ConvPlan pl;
  conv_plan(d, 0, mode, c, &pl);
  const cudaStream_t st = as_stream(stream);
  double* const fused = pl.fused_stats ? stats : nullptr;
  switch (pl.family) {
    case CONV_TC_3X3: case CONV_TC_1X1: case CONV_TC_1X1_S2:
      rc = conv_fwd_tc(pl, d, x, aux->w_t, aux->w_t_lo, bias, residual, y, relu, fused, st);
      break;
    case CONV_TC_ODD_3X3: rc = conv_fwd_odd_tc(pl, x, aux->w_t, aux->w_t_lo, bias, residual, y, relu, st); break;
    default: rc = conv_fwd_simt(pl, d, x, w, bias, residual, y, relu, fused, st); break;
  }
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
  if ((rc = ensure_setup())) return rc;
  ConvCall c;
  c.w_lo = aux && aux->w_lo;
  c.beta = beta;
  c.sms = sm_count();
  ConvPlan pl;
  const cudaStream_t st = as_stream(stream);
  switch (conv_plan(d, 1, mode, c, &pl)) {
    case CONV_TC_3X3: case CONV_TC_1X1: case CONV_TC_1X1_S2: case CONV_TC_DGRAD_3X3S2:
      return conv_dgrad_tc(pl, d, dy, w, c.w_lo ? aux->w_lo : nullptr, dx, beta, st);
    case CONV_TC_ODD_3X3: return conv_dgrad_odd_tc(pl, dy, w, c.w_lo ? aux->w_lo : nullptr, dx, beta, st);
    default: return conv_dgrad_simt(pl, d, dy, w, dx, beta, st);
  }
}
extern "C" int se_conv2d_dgrad(const se_conv_desc* d, const float* dy, const float* w, float* dx, float beta, int mode,
                               void* stream) {
  return se_conv2d_dgrad_aux(d, dy, w, nullptr, dx, beta, mode, stream);
}

// The kernel a plan launches, as torch.profiler names it: its demangled signature without the return type
static void kernel_name(const ConvPlan& pl, int dir, char* out, size_t n) {
  const SimtParams& f = pl.fp;
  const char* tile = f.bn == 16 ? "128, 16, 4, 2" : f.bn == 32 ? "128, 32, 4, 4" : "64, 64, 4, 4";
  const char* simt_w = "(se::ConvP, float const*, float const*, float*, float*, int, int, int, int)";
  switch (pl.family) {
    case CONV_FP32_TILES:
      snprintf(out, n, dir ? "se::conv_dgrad_kernel<%s, %s>(se::ConvP, float const*, float const*, float*, float, int)"
                           : "se::conv_fwd_kernel<%s, %s>(se::ConvP, float const*, float const*, float const*, float const*, "
                             "float*, int, double*)", tile, f.vec ? "true" : "false");
      break;
    case CONV_FP32_DENSE_SMALL:
      snprintf(out, n, "se::dense_small_fwd_kernel(float const*, float const*, float const*, float*, int, int, int, int)");
      break;
    case CONV_FP32_FWD_STEM:
      snprintf(out, n, "se::conv_fwd_stem_kernel(se::ConvP, float const*, float const*, float const*, float*, int, double*, int)");
      break;
    case CONV_FP32_WGRAD:
      snprintf(out, n, "se::conv_wgrad_kernel<64, 64, 4, 4>(se::ConvP, float const*, float const*, float*, float*, long long, int)");
      break;
    case CONV_FP32_WGRAD_STEM: snprintf(out, n, "se::conv_wgrad_stem_kernel%s", simt_w); break;
    case CONV_FP32_WGRAD_3X3: snprintf(out, n, "se::conv_wgrad3x3_kernel<%d, %d>%s", f.nci, f.nco, simt_w); break;
    case CONV_TC_WGRAD:
      snprintf(out, n, "se::conv_wgrad_tc_kernel<%d, %d, %d>(float const*, float const*, se::WgTcParams%s)", pl.wg_bn, pl.x3,
               pl.wg_np, pl.wg.box_tiles ? ", se::WgBox" : "");
      break;
    case CONV_TC_ODD_3X3:
      snprintf(out, n, dir == 2 ? "se::conv_odd_wgrad_tc_kernel<%d, %d>(float const*, float const*, se::OddWgParams)"
                                : "se::conv_odd_tc_kernel<%d, %d>(float const*, float const*, float const*, se::OddTcParams)",
               pl.od_bn, pl.x3);
      break;
    default:
      snprintf(out, n, "se::conv_tc_kernel<%d, %d, %d>(CUtensorMap_st, CUtensorMap_st, CUtensorMap_st, se::ConvTcParams)",
               pl.tc.BN, pl.x3, pl.tc.cblk / 8);
  }
}

extern "C" int se_conv2d_plan(const se_conv_desc* d, int mode, int direction, int sms, se_conv_plan_info* info) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(direction >= 0 && direction <= 2, "direction: 0 forward, 1 backward data, 2 weight gradient");
  SE_REQUIRE(info && sms >= 0, "bad arguments");
  ConvCall c;
  c.sms = sms;
  ConvPlan pl;
  conv_plan(d, direction, mode, c, &pl);
  const long long T = (long long)d->kh * d->kw * d->Cin * d->Cout;
  info->tensor_core = conv_is_tc(pl.family);
  info->splits = pl.splits;
  info->workspace = direction == 2 && pl.splits * (T + d->Cout) <= WG_WS_FLOATS;
  info->split_px = pl.split_px;
  kernel_name(pl, direction, info->kernel, sizeof(info->kernel));
  return SE_OK;
}

extern "C" int se_conv2d_path(const se_conv_desc* d, int mode, int direction) {
  se_conv_plan_info info;
  const int rc = se_conv2d_plan(d, mode, direction, 0, &info);
  return rc ? rc : info.tensor_core;
}

extern "C" int se_conv2d_wgrad(const se_conv_desc* d, const float* x, const float* dy, float* dw, float* dbias, int mode,
                               void* stream) {
  int rc = check_desc(d);
  if (rc) return rc;
  SE_REQUIRE(x && dy && dw, "null pointer");
  if ((rc = ensure_setup())) return rc;
  ConvCall c;
  c.aligned = aligned16(dw) && aligned16(dbias);    // the tensor-core kernels store dW / dbias as float2 / float4
  c.dy_aligned = aligned16(dy);
  c.sms = sm_count();
  ConvPlan pl;
  conv_plan(d, 2, mode, c, &pl);
  // Split-K: the kernel writes its partial sums into pl.splits slices of the workspace, and wgrad_reduce adds them into
  // dW / dbias in slice order; when they do not fit, the kernel adds them itself with atomics (direct mode)
  const cudaStream_t st = as_stream(stream);
  const long long T = (long long)d->kh * d->kw * d->Cin * d->Cout;
  float* ws = nullptr;
  if ((rc = wgrad_workspace(pl.splits * (T + d->Cout), st, &ws))) return rc;
  const WgOut o = ws ? WgOut{ws, ws, dbias ? ws + pl.splits * T : nullptr} : WgOut{nullptr, dw, dbias};
  switch (pl.family) {
    case CONV_TC_WGRAD: rc = conv_wgrad_tc(pl, x, dy, o, st); break;
    case CONV_TC_ODD_3X3: rc = conv_wgrad_odd_tc(pl, x, dy, o, st); break;
    default: rc = conv_wgrad_simt(pl, d, x, dy, o, st); break;
  }
  return (rc || !ws) ? rc : wgrad_reduce(ws, (int)pl.splits, T, d->Cout, dw, dbias, st);
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

namespace se {
cudaStream_t comm_stream();
cudaEvent_t comm_event();
bool comm_ready();
int comm_allreduce_ranges(float* base, const long long* off, const long long* cnt, int nranges, cudaStream_t st);
}

// `waiter` waits for the work issued so far on `st`
static void wait_for(cudaStream_t waiter, cudaStream_t st, cudaEvent_t ev) {
  cudaEventRecord(ev, st);
  cudaStreamWaitEvent(waiter, ev, 0);
}

// The stream ordering of one se_run_ops call.  Besides the caller's (main) stream a multi-op plan uses two branches:
// the side stream (weight gradients, and the filter transposition at the start of a step) and the communication stream
// (all-reduces).  These joins are what keeps the optimizer from racing the gradient writes, so the rule is:
//   - an op that reads or clears gradient memory -- MEMSET with i[0] bit 0 set, SGD_PREPARE, SGD_APPLY, ADAGRAD_APPLY --
//     first joins both branches;
//   - the first CONV_FWD / CONV_BN_FWD that reads a transposed filter joins the transposition;
//   - an ALLREDUCE waits for the main stream, and for the side stream when that branch is open;
//   - the end of the call joins everything, on every path (an unjoined fork would invalidate an ongoing capture).
struct Streams {
  cudaStream_t main;
  const se_runner* r;
  bool use_side;              // a multi-op plan, or any plan of a runner of its own
  bool side_open = false;     // side-stream work not yet joined
  bool transposing = false;   // ... and it is the filter transposition
  bool comm_pending = false;  // all-reduces not yet joined

  cudaStream_t fork_side() {
    if (!use_side) return main;
    wait_for(r->side, main, r->ev_fork);
    side_open = true;
    return r->side;
  }
  void join_side() {
    if (!side_open) return;
    wait_for(main, r->side, r->ev_join);
    side_open = transposing = false;
  }
  cudaStream_t fork_comm() {
    const cudaStream_t cs = comm_stream();
    wait_for(cs, main, comm_event());
    if (side_open) wait_for(cs, r->side, comm_event());
    comm_pending = true;
    return cs;
  }
  void join_comm() {
    if (!comm_pending) return;
    wait_for(main, comm_stream(), comm_event());
    comm_pending = false;
  }
  void join_all() {
    join_comm();
    join_side();
  }
};

// the arithmetic mode of a convolution op: its own (i[13] >= 0) or the plan's
static int op_mode(const int32_t* i, int mode) { return i[13] >= 0 ? i[13] : mode; }

static int run_ops_impl(const se_op* ops, int n, int mode, void* stream, Streams& st);

extern "C" int se_run_ops(const se_op* ops, int n, int mode, void* stream) {
  SE_REQUIRE(ops && n >= 0, "bad arguments");
  int rc = ensure_setup();
  if (rc) return rc;
  Streams st{as_stream(stream), &g_default_runner, n > 1};
  rc = run_ops_impl(ops, n, mode, stream, st);
  st.join_all();
  return rc;
}

extern "C" int se_runner_create(void** runner) {
  SE_REQUIRE(runner, "null pointer");
  *runner = nullptr;
  int rc = ensure_setup();
  if (rc) return rc;
  se_runner* r = new se_runner();
  if ((rc = runner_init(r))) {
    delete r;
    return rc;
  }
  *runner = r;
  return SE_OK;
}

extern "C" int se_runner_destroy(void* runner) {
  if (!runner) return SE_OK;
  SE_REQUIRE(runner != &g_default_runner, "the default runner belongs to the library");
  se_runner* r = static_cast<se_runner*>(runner);
  runner_free(r);
  delete r;
  return SE_OK;
}

// Plans that run at the same time -- CUDA graphs captured from them and replayed on different streams -- must not share a
// side stream: the side stream names the split-K workspace of their weight gradients.  A runner's side stream is its own,
// so its plans write their own workspace; the workspace has the default runner's size, so every split plan, and every
// bit, is the same on any runner.  Two more rules keep concurrent plans apart:
//   - the BatchNorm kernels with a grid-wide barrier are launched cooperatively: their CTAs are co-resident only if the
//     grid is launched as a whole, which another plan's kernels holding SMs (another such barrier above all) do not
//     otherwise guarantee.  The kernels, grids and results are the same; only the programmatic dependent launch of those
//     kernels is lost;
//   - the communication stream is process-wide, so a runner refuses plans with SE_OP_ALLREDUCE.
extern "C" int se_run_ops_runner(const se_op* ops, int n, int mode, void* stream, void* runner) {
  SE_REQUIRE(ops && n >= 0 && runner, "bad arguments");
  for (int k = 0; k < n; ++k)
    if (ops[k].opcode == SE_OP_ALLREDUCE) {
      set_error("se_run_ops_runner: SE_OP_ALLREDUCE at index %d: all-reduces run on the process-wide communication "
                "stream, with se_run_ops only", k);
      return SE_ERR_ARG;
    }
  int rc = ensure_setup();
  if (rc) return rc;
  Streams st{as_stream(stream), static_cast<const se_runner*>(runner), true};
  t_runner_plan = true;
  rc = run_ops_impl(ops, n, mode, stream, st);
  t_runner_plan = false;
  st.join_all();
  return rc;
}

static int run_ops_impl(const se_op* ops, int n, int mode, void* stream, Streams& st) {
  for (int k = 0; k < n; ++k) {
    const se_op& o = ops[k];
    const int32_t* i = o.i;
    const float* f = o.f;
    void* const* p = o.p;
    int rc = SE_OK;
    switch (o.opcode) {
      case SE_OP_CONV_FWD: {
        se_conv_desc d = desc_from(i);
        if (st.transposing && p[6]) st.join_side();
        se_conv_aux aux = {(const float*)p[6], (const float*)p[7], nullptr};
        rc = se_conv2d_fwd_aux(&d, (const float*)p[0], (const float*)p[1], &aux, (const float*)p[2],
                               (const float*)p[3], (float*)p[4], i[12], (double*)p[5], op_mode(i, mode), stream);
        break;
      }
      case SE_OP_CONV_BN_FWD: {
        // p: 0 x, 1 w, 2 bias, 3 y, 4 stats, 5 w_t, 6 gamma, 7 beta, 8 moving_mean, 9 moving_var, 10 save_mean,
        //    11 save_invstd, 12 residual, 13 bn_out, 14 counter;  i[12] conv relu, i[14] bn relu;  f: eps, momentum
        se_conv_desc d = desc_from(i);
        if (st.transposing && p[5]) st.join_side();
        rc = se_conv_bn_fwd(&d, (const float*)p[0], (const float*)p[1], (const float*)p[5], (const float*)p[2], (float*)p[3],
                            i[12], (double*)p[4], (const float*)p[6], (const float*)p[7], f[0], f[1], (float*)p[8],
                            (float*)p[9], (float*)p[10], (float*)p[11], (const float*)p[12], i[14], (float*)p[13], p[14],
                            op_mode(i, mode), stream);
        break;
      }
      case SE_OP_CONV_DGRAD: {
        se_conv_desc d = desc_from(i);
        se_conv_aux aux = {nullptr, nullptr, (const float*)p[3]};
        rc = se_conv2d_dgrad_aux(&d, (const float*)p[0], (const float*)p[1], &aux, (float*)p[2], f[0], op_mode(i, mode),
                                 stream);
        break;
      }
      case SE_OP_CONV_WGRAD: {
        se_conv_desc d = desc_from(i);
        rc = se_conv2d_wgrad(&d, (const float*)p[0], (const float*)p[1], (float*)p[2], (float*)p[3], op_mode(i, mode),
                             st.fork_side());
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
        if (i[0] & 1) st.join_all();   // gradient memory (frozen parameters, Engine.set_trainable)
        cudaError_t e = cudaMemsetAsync(p[0], 0, (size_t)(uintptr_t)p[1], as_stream(stream));
        if (e != cudaSuccess) { set_error("memset: %s", cudaGetErrorString(e)); rc = SE_ERR_CUDA; }
        break;
      }
      case SE_OP_TRANSPOSE_FILTERS:
        if (mode == SE_MODE_TF32 || mode == SE_MODE_TF32X3) {
          // the transposed filter copies are first needed by the first tensor-core convolution: the transposition runs
          // on the side stream beside the statistics memset, the stem convolution and its BatchNorm
          cudaStream_t ts = st.main;
          if (!st.side_open) {
            ts = st.fork_side();
            st.transposing = st.side_open;
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
        if (!se::comm_ready()) { set_error("SE_OP_ALLREDUCE without a communicator (se_comm_init)"); return SE_ERR_ARG; }
        long long off[7], cnt[7];
        const int nr = i[0] < 7 ? i[0] : 7;
        for (int r = 0; r < nr; ++r) { off[r] = (long long)(uintptr_t)p[1 + 2 * r]; cnt[r] = (long long)(uintptr_t)p[2 + 2 * r]; }
        rc = se::comm_allreduce_ranges((float*)p[0], off, cnt, nr, st.fork_comm());
        break;
      }
      case SE_OP_SGD_PREPARE:
        st.join_all();
        rc = se_sgd_prepare((const float*)p[0], (float*)p[1], (int64_t)(uintptr_t)p[2], (const se_l2_segment*)p[3], i[0],
                            (double*)p[4], stream);
        break;
      case SE_OP_SGD_APPLY:
        st.join_all();
        // p[3] = lr_state {lr, decay, iterations, lr_t}: the schedule kernel derives this step's lr_t, the update reads it
        rc = se_sgd_schedule((float*)p[3], stream);
        if (rc == SE_OK)
          rc = se_sgd_apply_devlr((float*)p[0], (const float*)p[1], (float*)p[5], (int64_t)(uintptr_t)p[2],
                                  (const float*)p[3] + 3, f[0], i[0], f[1], (const double*)p[4], stream);
        break;
      case SE_OP_ADAGRAD_APPLY:
        // the Adagrad update in place of SGD_APPLY: same p[0..5] (p[5] = accumulators), f[0] = epsilon, f[1] = clipnorm
        st.join_all();
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
