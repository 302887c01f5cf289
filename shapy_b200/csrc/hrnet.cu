// HRNet-W48 executor: a flat program of STEM / CONV / FUSE / POOL ops over numbered NHWC activation
// slots (built by the Python host mirror from the reference module tree,
// regressor/human_shape/models/backbone/hrnet.py:202-498), run as a fixed sequence of launches with no
// host synchronisation, so it can be captured in a CUDA graph.
//   create : folds BatchNorm into the conv weights (scale) and a per-channel bias (shift), packs the
//            weights as [tap][cout][cin] fp16 hi/lo planes on the device.
//   bind   : (first forward for a given workspace / batch / image size) lays the slots out in the
//            caller's workspace and encodes the TMA descriptors of every wgmma convolution.
//   forward: ~380 launches (331 convs + fuse sums + pool) instead of the reference's ~1100.
#include <array>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "conv.cuh"

using namespace shapy;

struct shapy_hrnet {
  std::vector<ConvW> convs;
  std::vector<shapy_op_t> ops;
  std::vector<shapy_slot_t> slots;
  int feat_slot = -1, mode = 1, engine = 0;
  std::vector<void *> allocs;
  // binding
  void *ws = nullptr;
  int B = 0, H = 0, W = 0;
  std::vector<ActView> views;
  std::vector<WgmmaPlan *> plans;  // per op (null when the op does not use the wgmma engine)
  // lane schedule (built by bind): lane 0 is the caller's stream, lanes 1.. are streams owned by this object
  int n_lanes = 1;
  int device = -1;
  cudaStream_t lane_stream[SHAPY_MAX_LANES] = {nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t fork_ev = nullptr, join_ev[SHAPY_MAX_LANES] = {nullptr, nullptr, nullptr, nullptr};
  std::vector<cudaEvent_t> op_ev;            // per op: recorded after the op when an op of another lane waits on it
  std::vector<std::vector<int>> op_waits;    // per op: ops of other lanes to wait for (transitively reduced)
  std::vector<char> op_pdl;                  // per op: programmatic dependent launch allowed (no other lane can be running)
  // CUDA graph of one forward (captured on the second forward after a bind, replayed afterwards): the stem and the
  // pool read the image / feature pointers from `io_cells`, so one graph serves any input and output buffer
  void **io_cells = nullptr;                 // device: [0] = images, [1] = feats
  cudaStream_t cap_stream = nullptr;         // capture origin (the caller's stream may be the legacy default stream)
  cudaGraphExec_t graph_exec = nullptr;
  long long graph_kernels = 0;
  bool warm = false, graph_failed = false;
};

static void free_plans(shapy_hrnet *p) {
  if (p->graph_exec) cudaGraphExecDestroy(p->graph_exec);
  p->graph_exec = nullptr; p->graph_kernels = 0; p->warm = false; p->graph_failed = false;
  for (auto *u : p->plans) if (u) wgmma_plan_destroy(u);
  p->plans.clear();
  for (auto e : p->op_ev) if (e) cudaEventDestroy(e);
  p->op_ev.clear();
  p->op_waits.clear();
  p->op_pdl.clear();
}

static void free_lanes(shapy_hrnet *p) {
  for (int l = 1; l < SHAPY_MAX_LANES; ++l) {
    if (p->lane_stream[l]) cudaStreamDestroy(p->lane_stream[l]);
    if (p->join_ev[l]) cudaEventDestroy(p->join_ev[l]);
    p->lane_stream[l] = nullptr; p->join_ev[l] = nullptr;
  }
  if (p->fork_ev) cudaEventDestroy(p->fork_ev);
  p->fork_ev = nullptr;
  if (p->cap_stream) cudaStreamDestroy(p->cap_stream);
  p->cap_stream = nullptr;
  if (p->io_cells) cudaFree(p->io_cells);
  p->io_cells = nullptr;
}

// ---------------------------------------------------------------------------------------------------------------
// Lane schedule.  The independent branches of a HighResolutionModule (reference hrnet.py:175-193), the (i, j) convs
// of its fuse stage and the down-sample convs of the bottlenecks are given different lanes by the host mirror; here
// every ordering between lanes is derived from the slots (and channel ranges) the ops read and write in PROGRAM
// order -- RAW, WAR and WAW, so liveness-based slot reuse stays correct -- and reduced with vector clocks to the
// cross-stream event waits that are really needed.  Persistent kernels of different lanes then back-fill each
// other's tails: 896 equal work items on 132 SMs are 7 rounds of 6.8, 196 tiles 2 rounds of 1.48.
struct Access { int slot, c0, c1; bool write; };

static void op_accesses(const shapy_hrnet *p, const shapy_op_t &o, std::vector<Access> &acc) {
  acc.clear();
  auto whole = [&](int s, bool w) { acc.push_back({s, 0, p->slots[s].channels, w}); };
  switch (o.kind) {
    case SHAPY_OP_STEM: {
      const ConvW &w = p->convs[o.conv];
      acc.push_back({o.out_slot, o.out_coff, o.out_coff + w.cout, true});
      break;
    }
    case SHAPY_OP_CONV: {
      const ConvW &w = p->convs[o.conv];
      acc.push_back({o.in_slot, 0, w.cin, false});
      if (o.res_slot >= 0) acc.push_back({o.res_slot, 0, w.cout, false});
      acc.push_back({o.out_slot, o.out_coff, o.out_coff + w.cout, true});
      break;
    }
    case SHAPY_OP_FUSE: {
      const int C = p->slots[o.fuse_in[0]].channels;
      for (int k = 0; k < o.n_in; ++k) whole(o.fuse_in[k], false);
      acc.push_back({o.out_slot, o.out_coff, o.out_coff + C, true});
      break;
    }
    case SHAPY_OP_POOL: whole(o.in_slot, false); break;
    default: break;
  }
}

static int max_lanes() {
  static int v = -1;
  if (v < 0) { const char *e = getenv("SHAPY_HRNET_LANES"); v = e ? std::max(1, std::min(atoi(e), (int)SHAPY_MAX_LANES)) : SHAPY_MAX_LANES; }
  return v;
}
// SHAPY_PDL: 0 never, 1 (default) every conv launch, 2 only where no other lane can be running.  The default lets the
// early-launched dependent's prologue overlap its predecessor's tail.
static int pdl_policy() {
  static int v = -1;
  if (v < 0) { const char *e = getenv("SHAPY_PDL"); v = e ? atoi(e) : 1; }
  return v;
}

static int lane_of(const shapy_op_t &o) { return std::max(0, std::min(o.lane, max_lanes() - 1)); }

static int build_schedule(shapy_hrnet *p) {
  const int n = (int)p->ops.size();
  p->op_waits.assign(n, {});
  p->op_pdl.assign(n, 1);
  p->op_ev.assign(n, nullptr);
  p->n_lanes = 1;
  for (auto &o : p->ops) p->n_lanes = std::max(p->n_lanes, lane_of(o) + 1);
  if (!p->fork_ev) SHAPY_CUDA_TRY(cudaEventCreateWithFlags(&p->fork_ev, cudaEventDisableTiming));
  for (int l = 1; l < p->n_lanes; ++l) {
    if (!p->lane_stream[l]) SHAPY_CUDA_TRY(cudaStreamCreateWithFlags(&p->lane_stream[l], cudaStreamNonBlocking));
    if (!p->join_ev[l]) SHAPY_CUDA_TRY(cudaEventCreateWithFlags(&p->join_ev[l], cudaEventDisableTiming));
  }
  std::vector<std::vector<Access>> acc(n);
  for (int i = 0; i < n; ++i) op_accesses(p, p->ops[i], acc[i]);
  // vc[i][m]: the latest op of lane m that is ordered before (or is) op i
  std::vector<std::array<int, SHAPY_MAX_LANES>> vc(n);
  int last_in_lane[SHAPY_MAX_LANES] = {-1, -1, -1, -1};
  std::vector<char> need_ev(n, 0);
  for (int i = 0; i < n; ++i) {
    const int L = lane_of(p->ops[i]);
    std::array<int, SHAPY_MAX_LANES> c;
    if (last_in_lane[L] >= 0) c = vc[last_in_lane[L]]; else c.fill(-1);
    // conflicting earlier ops of other lanes, latest first (a later one usually subsumes the earlier ones)
    for (int j = i - 1; j >= 0; --j) {
      const int M = lane_of(p->ops[j]);
      if (M == L || j <= c[M]) continue;
      bool conflict = false;
      for (const Access &a : acc[i]) {
        for (const Access &b : acc[j])
          if (a.slot == b.slot && (a.write || b.write) && a.c0 < b.c1 && b.c0 < a.c1) { conflict = true; break; }
        if (conflict) break;
      }
      if (!conflict) continue;
      p->op_waits[i].push_back(j);
      need_ev[j] = 1;
      for (int m = 0; m < SHAPY_MAX_LANES; ++m) c[m] = std::max(c[m], vc[j][m]);
    }
    c[L] = i;
    vc[i] = c;
    last_in_lane[L] = i;
  }
  for (int i = 0; i < n; ++i)
    if (need_ev[i]) SHAPY_CUDA_TRY(cudaEventCreateWithFlags(&p->op_ev[i], cudaEventDisableTiming));
  // PDL only where nothing of another lane can run concurrently with the op (see pdl_policy)
  const int pol = pdl_policy();
  int n_conc = 0, n_waits = 0;
  for (int i = 0; i < n; ++i) {
    const int L = lane_of(p->ops[i]);
    bool conc = false;
    for (int j = 0; j < n && !conc; ++j) {
      const int M = lane_of(p->ops[j]);
      if (M == L) continue;
      const bool j_before_i = vc[i][M] >= j, i_before_j = vc[j][L] >= i;
      if (!j_before_i && !i_before_j) conc = true;
    }
    p->op_pdl[i] = pol == 0 ? 0 : (pol == 1 ? 1 : (conc || !p->op_waits[i].empty() ? 0 : 1));
    n_conc += conc;
    n_waits += (int)p->op_waits[i].size();
  }
  if (getenv("SHAPY_CONV_DEBUG"))
    fprintf(stderr, "[hrnet] schedule: %d ops, %d lanes, %d ops with a concurrent lane, %d cross-lane waits\n", n, p->n_lanes,
            n_conc, n_waits);
  return SHAPY_OK;
}

template <typename T>
static T *dev_upload(std::vector<void *> &allocs, const std::vector<T> &h, cudaError_t &err) {
  T *d = nullptr;
  if (err != cudaSuccess) return nullptr;
  err = cudaMalloc((void **)&d, std::max<size_t>(h.size(), 1) * sizeof(T));
  if (err != cudaSuccess) return nullptr;
  allocs.push_back(d);
  if (!h.empty()) err = cudaMemcpy(d, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice);
  return d;
}

// Folds BN and packs one conv.  Returns false on CUDA failure.
static bool pack_conv(const shapy_conv_desc_t &c, bool stem, ConvW &out, std::vector<void *> &allocs, cudaError_t &err) {
  const int taps = c.ksize * c.ksize;
  std::vector<float> scale(c.cout, 1.f), bias(c.cout, 0.f);
  for (int o = 0; o < c.cout; ++o) {
    float b = c.bias ? c.bias[o] : 0.f;
    if (c.bn_weight) {
      // y = (conv + b - mean) * gamma / sqrt(var + eps) + beta   (eval-mode BatchNorm2d)
      float s = c.bn_weight[o] / std::sqrt(c.bn_var[o] + c.bn_eps);
      scale[o] = s;
      bias[o] = (b - c.bn_mean[o]) * s + c.bn_bias[o];
    } else {
      bias[o] = b;
    }
  }
  out.cin = c.cin; out.cout = c.cout; out.ksize = c.ksize; out.stride = c.stride;
  out.bias = dev_upload(allocs, bias, err);
  if (stem) {
    std::vector<float> wf((size_t)taps * c.cin * c.cout);
    for (int o = 0; o < c.cout; ++o)
      for (int i = 0; i < c.cin; ++i)
        for (int t = 0; t < taps; ++t)
          wf[((size_t)t * c.cin + i) * c.cout + o] = c.weight[((size_t)o * c.cin + i) * taps + t] * scale[o];
    out.w_f32 = dev_upload(allocs, wf, err);
    return err == cudaSuccess;
  }
  std::vector<__half> hi((size_t)taps * c.cout * c.cin), lo(hi.size());
  for (int o = 0; o < c.cout; ++o)
    for (int i = 0; i < c.cin; ++i)
      for (int t = 0; t < taps; ++t) {
        float v = c.weight[((size_t)o * c.cin + i) * taps + t] * scale[o];
        __half h = __float2half_rn(v);
        size_t d = ((size_t)t * c.cout + o) * c.cin + i;
        hi[d] = h;
        lo[d] = __float2half_rn((v - __half2float(h)) * kLoScale);
      }
  out.w_hi = dev_upload(allocs, hi, err);
  out.w_lo = dev_upload(allocs, lo, err);
  return err == cudaSuccess;
}

extern "C" int shapy_hrnet_create(shapy_hrnet_t **out, const shapy_conv_desc_t *convs, int n_convs,
                                  const shapy_op_t *ops, int n_ops, const shapy_slot_t *slots, int n_slots,
                                  int feat_slot, int mode, int engine) {
  SHAPY_REQUIRE(out && convs && ops && slots && n_convs > 0 && n_ops > 0 && n_slots > 0, "shapy_hrnet_create: bad argument");
  SHAPY_REQUIRE(mode == 0 || mode == 1, "shapy_hrnet_create: mode %d", mode);
  auto *p = new shapy_hrnet();
  p->ops.assign(ops, ops + n_ops);
  p->slots.assign(slots, slots + n_slots);
  p->feat_slot = feat_slot; p->mode = mode; p->engine = engine;
  std::vector<char> is_stem(n_convs, 0);
  for (auto &o : p->ops) {
    if ((o.kind == SHAPY_OP_STEM || o.kind == SHAPY_OP_CONV) && (o.conv < 0 || o.conv >= n_convs)) {
      delete p; set_error("op references conv %d of %d", o.conv, n_convs); return SHAPY_ERR_ARG;
    }
    if (o.kind == SHAPY_OP_STEM) is_stem[o.conv] = 1;
  }
  cudaError_t err = cudaSuccess;
  p->convs.resize(n_convs);
  for (int i = 0; i < n_convs; ++i) {
    if (!pack_conv(convs[i], is_stem[i], p->convs[i], p->allocs, err)) break;
  }
  if (err != cudaSuccess) {
    set_error("shapy_hrnet_create: %s", cudaGetErrorString(err));
    shapy_hrnet_destroy(p);
    return (int)err;
  }
  *out = p;
  return SHAPY_OK;
}

extern "C" void shapy_hrnet_destroy(shapy_hrnet_t *p) {
  if (!p) return;
  free_plans(p);
  free_lanes(p);
  for (void *a : p->allocs) cudaFree(a);
  delete p;
}

static size_t slot_bytes(const shapy_hrnet *p, int s, int B, int H, int W) {
  const shapy_slot_t &sl = p->slots[s];
  size_t plane = (size_t)B * (H / sl.div) * (W / sl.div) * sl.channels * sizeof(__half);
  return align_up(plane, 1024) * (p->mode ? 2 : 1);
}

extern "C" size_t shapy_hrnet_workspace_bytes(const shapy_hrnet_t *p, int B, int H, int W) {
  if (!p || B <= 0 || H % 32 || W % 32) return 0;
  size_t total = 1024;
  for (size_t s = 0; s < p->slots.size(); ++s) total += slot_bytes(p, (int)s, B, H, W);
  return total;
}

static ActView view_of(const shapy_hrnet *p, int slot, int coff, int C) {
  ActView v = p->views[slot];
  v.coff = coff;
  v.C = C;
  return v;
}

static int bind(shapy_hrnet *p, void *ws, int B, int H, int W) {
  free_plans(p);
  p->views.assign(p->slots.size(), ActView());
  char *base = (char *)(((uintptr_t)ws + 1023) & ~(uintptr_t)1023);
  for (size_t s = 0; s < p->slots.size(); ++s) {
    const shapy_slot_t &sl = p->slots[s];
    ActView &v = p->views[s];
    v.N = B; v.H = H / sl.div; v.W = W / sl.div; v.C = sl.channels; v.Ctot = sl.channels; v.coff = 0;
    size_t plane = align_up((size_t)B * v.H * v.W * sl.channels * sizeof(__half), 1024);
    v.hi = (__half *)base;
    v.lo = p->mode ? (__half *)(base + plane) : nullptr;
    base += plane * (p->mode ? 2 : 1);
  }
  p->plans.assign(p->ops.size(), nullptr);
  for (size_t i = 0; i < p->ops.size(); ++i) {
    const shapy_op_t &o = p->ops[i];
    if (o.kind != SHAPY_OP_CONV || p->engine == 1) continue;
    const ConvW &w = p->convs[o.conv];
    ActView in = view_of(p, o.in_slot, 0, w.cin), out = view_of(p, o.out_slot, o.out_coff, w.cout);
    ActView res;
    if (o.res_slot >= 0) res = view_of(p, o.res_slot, 0, w.cout);
    if (!wgmma_supported(w, in, out)) continue;  // falls back to the SIMT engine for this layer
    p->plans[i] = wgmma_plan_create(w, in, out, o.res_slot >= 0 ? &res : nullptr, o.relu != 0);
    if (!p->plans[i]) return SHAPY_ERR_STATE;
  }
  int rc = build_schedule(p);
  if (rc) return rc;
  p->ws = ws; p->B = B; p->H = H; p->W = W;
  return SHAPY_OK;
}

// Enqueues one forward on `st` (+ the lane streams).  cells != null: the stem / pool read their buffers from the device
// cells (graph capture); `images` then only conveys the alignment of the future inputs.
// SHAPY_HRNET_TRACE=<file>: the direct path records a start / end event pair around every op on its lane stream and
// shapy_hrnet_forward() dumps "op lane kind cin cout k s div start_us end_us" per op after a device synchronise
// (a debugging aid: the events add a little serialisation; never active under graph capture).
struct TraceEv { cudaEvent_t a, b; };
static std::vector<TraceEv> g_trace;
static cudaEvent_t g_trace0 = nullptr;
static const char *trace_path() {
  static const char *v = getenv("SHAPY_HRNET_TRACE");
  return v;
}

static int enqueue_forward(shapy_hrnet *p, const float *images, float *feats, void **cells, int B, int H, int W,
                           cudaStream_t st) {
  const bool trace = trace_path() && !cells;
  if (trace) {
    if (g_trace.size() != p->ops.size()) {
      g_trace.resize(p->ops.size());
      for (auto &t : g_trace) { cudaEventCreate(&t.a); cudaEventCreate(&t.b); }
      cudaEventCreate(&g_trace0);
    }
    cudaEventRecord(g_trace0, st);
  }
  // fork: the other lanes start after everything already queued on the caller's stream (the input images, and the
  // join of the previous forward on this workspace)
  p->lane_stream[0] = st;
  if (p->n_lanes > 1) {
    SHAPY_CUDA_TRY(cudaEventRecord(p->fork_ev, st));
    for (int l = 1; l < p->n_lanes; ++l) SHAPY_CUDA_TRY(cudaStreamWaitEvent(p->lane_stream[l], p->fork_ev, 0));
  }
  for (size_t i = 0; i < p->ops.size(); ++i) {
    const shapy_op_t &o = p->ops[i];
    cudaStream_t ls = p->lane_stream[lane_of(o)];
    for (int j : p->op_waits[i]) SHAPY_CUDA_TRY(cudaStreamWaitEvent(ls, p->op_ev[j], 0));
    if (trace) cudaEventRecord(g_trace[i].a, ls);
    int rc = SHAPY_OK;
    switch (o.kind) {
      case SHAPY_OP_STEM: {
        const ConvW &w = p->convs[o.conv];
        rc = launch_stem(w, images, cells ? (const float *const *)&cells[0] : nullptr, B, H, W,
                         view_of(p, o.out_slot, o.out_coff, w.cout), ls);
        break;
      }
      case SHAPY_OP_CONV: {
        const ConvW &w = p->convs[o.conv];
        if (p->plans[i]) {
          rc = wgmma_plan_launch(p->plans[i], ls, p->op_pdl[i] != 0);
        } else {
          ActView in = view_of(p, o.in_slot, 0, w.cin), out = view_of(p, o.out_slot, o.out_coff, w.cout), res;
          if (o.res_slot >= 0) res = view_of(p, o.res_slot, 0, w.cout);
          rc = launch_conv_simt(w, in, out, o.res_slot >= 0 ? &res : nullptr, o.relu != 0, ls);
        }
        break;
      }
      case SHAPY_OP_FUSE: {
        ActView ins[4];
        const int C = p->slots[o.fuse_in[0]].channels;  // may be a channel slice of a wider output slot
        for (int k = 0; k < o.n_in; ++k) ins[k] = view_of(p, o.fuse_in[k], 0, C);
        rc = launch_fuse(ins, o.fuse_shift, o.n_in, view_of(p, o.out_slot, o.out_coff, C), o.relu != 0, ls);
        break;
      }
      case SHAPY_OP_POOL:
        rc = launch_pool(p->views[o.in_slot], feats, cells ? (float *const *)&cells[1] : nullptr, ls);
        break;
      default:
        set_error("unknown op kind %d", o.kind);
        rc = SHAPY_ERR_ARG;
    }
    if (rc) return rc;
    if (trace) cudaEventRecord(g_trace[i].b, ls);
    if (p->op_ev[i]) SHAPY_CUDA_TRY(cudaEventRecord(p->op_ev[i], ls));
  }
  // join: the caller's stream continues after every lane has drained
  for (int l = 1; l < p->n_lanes; ++l) {
    SHAPY_CUDA_TRY(cudaEventRecord(p->join_ev[l], p->lane_stream[l]));
    SHAPY_CUDA_TRY(cudaStreamWaitEvent(st, p->join_ev[l], 0));
  }
  return SHAPY_OK;
}

static bool graph_enabled() {
  static int v = -1;
  if (v < 0) {
    const char *e = getenv("SHAPY_HRNET_GRAPH");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v == 1;
}

// Captures one forward (all lanes) into a CUDA graph.  Returns false (and leaves the direct path in charge) on any
// failure; never leaves a stream in capture mode.
static bool capture_graph(shapy_hrnet *p, const float *images, int B, int H, int W) {
  if (!p->cap_stream && cudaStreamCreateWithFlags(&p->cap_stream, cudaStreamNonBlocking) != cudaSuccess) return false;
  if (!p->io_cells && cudaMalloc((void **)&p->io_cells, 2 * sizeof(void *)) != cudaSuccess) return false;
  if (cudaStreamBeginCapture(p->cap_stream, cudaStreamCaptureModeThreadLocal) != cudaSuccess) { cudaGetLastError(); return false; }
  const long long n0 = shapy_launch_count();
  const int rc = enqueue_forward(p, images, nullptr, p->io_cells, B, H, W, p->cap_stream);
  cudaGraph_t g = nullptr;
  const cudaError_t e = cudaStreamEndCapture(p->cap_stream, &g);
  const long long n = shapy_launch_count() - n0;
  count_launch((int)-n);                      // nothing ran during the capture
  if (rc || e != cudaSuccess || !g) {
    if (g) cudaGraphDestroy(g);
    cudaGetLastError();
    return false;
  }
  cudaGraphExec_t ex = nullptr;
  const cudaError_t e2 = cudaGraphInstantiate(&ex, g, 0);
  cudaGraphDestroy(g);
  if (e2 != cudaSuccess) { cudaGetLastError(); return false; }
  p->graph_exec = ex;
  p->graph_kernels = n;
  if (getenv("SHAPY_CONV_DEBUG")) fprintf(stderr, "[hrnet] captured a CUDA graph with %lld kernel nodes\n", n);
  return true;
}

extern "C" int shapy_hrnet_forward(shapy_hrnet_t *p, const float *images, int B, int H, int W, float *feats,
                                   void *workspace, size_t workspace_bytes, void *stream) {
  SHAPY_REQUIRE(p && images && feats && workspace, "shapy_hrnet_forward: null argument");
  SHAPY_REQUIRE(B > 0 && H > 0 && W > 0 && H % 32 == 0 && W % 32 == 0, "shapy_hrnet_forward: image size %dx%d must be a multiple of 32", H, W);
  SHAPY_REQUIRE(workspace_bytes >= shapy_hrnet_workspace_bytes(p, B, H, W), "shapy_hrnet_forward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (p->ws != workspace || p->B != B || p->H != H || p->W != W) {
    int rc = bind(p, workspace, B, H, W);
    if (rc) return rc;
  }
  // CUDA graph replay: from the second forward of a binding on, unless the caller is itself capturing (then the direct
  // launches below simply become part of the caller's graph) or the input is not 16-byte aligned (the captured stem
  // kernel uses 128-bit loads)
  bool use_graph = graph_enabled() && !trace_path() && p->warm && !p->graph_failed && ((uintptr_t)images & 15) == 0;
  if (use_graph) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) { cudaGetLastError(); use_graph = false; }
  }
  if (use_graph && !p->graph_exec && !capture_graph(p, images, B, H, W)) { p->graph_failed = true; use_graph = false; }
  if (!use_graph) {
    int rc = enqueue_forward(p, images, feats, nullptr, B, H, W, st);
    p->warm = true;
    if (!rc && trace_path()) {
      cudaDeviceSynchronize();
      if (FILE *f = fopen(trace_path(), "w")) {
        for (size_t i = 0; i < p->ops.size(); ++i) {
          const shapy_op_t &o = p->ops[i];
          float t0 = 0, t1 = 0;
          cudaEventElapsedTime(&t0, g_trace0, g_trace[i].a);
          cudaEventElapsedTime(&t1, g_trace0, g_trace[i].b);
          const ConvW *w = (o.kind == SHAPY_OP_CONV || o.kind == SHAPY_OP_STEM) ? &p->convs[o.conv] : nullptr;
          fprintf(f, "%zu %d %d %d %d %d %d %d %.2f %.2f\n", i, lane_of(o), o.kind, w ? w->cin : 0, w ? w->cout : 0,
                  w ? w->ksize : 0, w ? w->stride : 0, p->slots[o.kind == SHAPY_OP_POOL ? o.in_slot : o.out_slot].div,
                  t0 * 1e3, t1 * 1e3);
        }
        fclose(f);
      }
    }
    return rc;
  }
  int rc = launch_set_io_cells(p->io_cells, images, feats, st);
  if (rc) return rc;
  SHAPY_CUDA_TRY(cudaGraphLaunch(p->graph_exec, st));
  count_launch((int)p->graph_kernels);
  return SHAPY_OK;
}

extern "C" int shapy_hrnet_read_slot(shapy_hrnet_t *p, int slot, float *dst, void *stream) {
  SHAPY_REQUIRE(p && dst && slot >= 0 && slot < (int)p->slots.size() && p->ws, "shapy_hrnet_read_slot: bad argument / not bound");
  return launch_nhwc_merge(p->views[slot], dst, true, (cudaStream_t)stream);
}

extern "C" double shapy_hrnet_flops(const shapy_hrnet_t *p, int B, int H, int W) {
  if (!p) return 0.0;
  double f = 0.0;
  for (auto &o : p->ops) {
    if (o.kind != SHAPY_OP_STEM && o.kind != SHAPY_OP_CONV) continue;
    const ConvW &w = p->convs[o.conv];
    const shapy_slot_t &so = p->slots[o.out_slot];
    f += 2.0 * B * (H / so.div) * (W / so.div) * w.cout * (double)w.cin * w.ksize * w.ksize;
  }
  return f;
}

// Standalone convolution on fp32 NHWC buffers (unit tests of both engines).
extern "C" int shapy_conv_test(const shapy_conv_desc_t *conv, const float *x, const float *res, int B, int H, int W,
                               int relu, int mode, int engine, float *y, void *stream) {
  SHAPY_REQUIRE(conv && x && y, "shapy_conv_test: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  std::vector<void *> allocs;
  cudaError_t err = cudaSuccess;
  ConvW w;
  int rc = SHAPY_OK;
  WgmmaPlan *plan = nullptr;
  auto cleanup = [&]() {
    cudaStreamSynchronize(st);
    if (plan) wgmma_plan_destroy(plan);
    for (void *a : allocs) cudaFree(a);
  };
  if (!pack_conv(*conv, false, w, allocs, err)) { cleanup(); set_error("conv_test: %s", cudaGetErrorString(err)); return (int)err; }
  const int Ho = conv->stride == 2 ? H / 2 : H, Wo = conv->stride == 2 ? W / 2 : W;
  auto make = [&](int n, int h, int ww, int c) {
    ActView v;
    v.N = n; v.H = h; v.W = ww; v.C = c; v.Ctot = c; v.coff = 0;
    size_t bytes = (size_t)n * h * ww * c * sizeof(__half);
    if (err == cudaSuccess) err = cudaMalloc((void **)&v.hi, bytes);
    if (err == cudaSuccess) allocs.push_back(v.hi);
    if (mode && err == cudaSuccess) { err = cudaMalloc((void **)&v.lo, bytes); if (err == cudaSuccess) allocs.push_back(v.lo); }
    return v;
  };
  ActView in = make(B, H, W, conv->cin), out = make(B, Ho, Wo, conv->cout), rv;
  if (res) rv = make(B, Ho, Wo, conv->cout);
  if (err != cudaSuccess) { cleanup(); set_error("conv_test: %s", cudaGetErrorString(err)); return (int)err; }
  if ((rc = launch_nhwc_split(x, in, st))) { cleanup(); return rc; }
  if (res && (rc = launch_nhwc_split(res, rv, st))) { cleanup(); return rc; }
  if (engine == 0) {
    plan = wgmma_plan_create(w, in, out, res ? &rv : nullptr, relu != 0);
    if (!plan) { cleanup(); return SHAPY_ERR_UNSUPPORTED; }
    rc = wgmma_plan_launch(plan, st, true);
    if (const char *reps_s = getenv("SHAPY_CONV_TEST_REPS")) {
      // timing aid for kernel work: re-launch the same plan and report the average launch time
      const int reps = atoi(reps_s);
      cudaEvent_t e0, e1;
      cudaEventCreate(&e0); cudaEventCreate(&e1);
      cudaEventRecord(e0, st);
      for (int i = 0; i < reps && !rc; ++i) rc = wgmma_plan_launch(plan, st, true);
      cudaEventRecord(e1, st);
      cudaStreamSynchronize(st);
      float ms = 0;
      cudaEventElapsedTime(&ms, e0, e1);
      const double fl = 2.0 * B * Ho * Wo * (double)conv->cout * conv->cin * conv->ksize * conv->ksize;
      fprintf(stderr, "[conv_test] cin %d cout %d k %d s %d %dx%d B %d mode %d: %.2f us/launch, %.1f TFLOP/s (x%d MMA flops)\n",
              conv->cin, conv->cout, conv->ksize, conv->stride, H, W, B, mode, ms * 1e3 / reps, fl / (ms * 1e-3 / reps) * 1e-12,
              mode ? 3 : 1);
      cudaEventDestroy(e0); cudaEventDestroy(e1);
    }
  } else {
    rc = launch_conv_simt(w, in, out, res ? &rv : nullptr, relu != 0, st);
  }
  if (!rc) rc = launch_nhwc_merge(out, y, false, st);
  cleanup();
  cudaError_t e2 = cudaGetLastError();
  if (!rc && e2 != cudaSuccess) { set_error("conv_test: %s", cudaGetErrorString(e2)); rc = (int)e2; }
  return rc;
}
