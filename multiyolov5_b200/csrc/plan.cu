// C ABI + layer-plan executor: what Model.__init__/fuse() and Model.forward_once (reference models/yolo.py:293-316,339-347)
// become on the device.  The host-side planner (multiyolov5_b200/plan.py) lowers the module tree to a flat op list over
// liveness-packed NHWC buffers; this file resolves views, owns packed weights / tensor maps and replays the list on a stream.
#include <nvtx3/nvToolsExt.h>
// NVTX ranges around every C-ABI entry point that launches work (SURVEY.md section 5): visible in nsys / ncu --nvtx, free when no tool is attached
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};
#include <stdarg.h>

#include <algorithm>
#include <string>
#include <vector>

#include "conv.h"
#include "kernels.h"
#include "train.h"

namespace myolo {

thread_local char g_err[1024] = "";
thread_local int64_t g_launch_count = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

static int check_device(int* sms) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) {
    set_error("no CUDA device: %s", cudaGetErrorString(e));
    return MYOLO_E_NODEVICE;
  }
  // cudaGetDeviceProperties costs milliseconds (and sometimes far more): query each device once
  static int cached_sms[64] = {};
  if (dev >= 0 && dev < 64 && cached_sms[dev] > 0) {
    if (sms) *sms = cached_sms[dev];
    return 0;
  }
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, dev);
  if (e != cudaSuccess) {
    set_error("cudaGetDeviceProperties: %s", cudaGetErrorString(e));
    return MYOLO_E_NODEVICE;
  }
  if (prop.major != 9 || prop.minor != 0) {
    set_error("libmyolo_sm90a needs an sm_90 (Hopper H100) device, found sm_%d%d (%s); there is no fallback path", prop.major,
              prop.minor, prop.name);
    return MYOLO_E_NODEVICE;
  }
  if (dev >= 0 && dev < 64) cached_sms[dev] = prop.multiProcessorCount;
  if (sms) *sms = prop.multiProcessorCount;
  return 0;
}

struct WeightSlot {
  __half* w = nullptr;
  float* bias = nullptr;
  int co = 0, ci = 0, k = 0, co_pad = 0, ci_pad = 0;
  bool set = false;
  // training
  const float* w_master = nullptr;   // caller's fp32 parameter (device)
  const float *gamma = nullptr, *beta = nullptr, *mean = nullptr, *var = nullptr, *bias_master = nullptr;   // as passed to set_conv_weights
  float eps = 0.f;
  float* d_w = nullptr;              // caller's .grad (accumulated)
  float* d_bias = nullptr;
  __half* w_dgrad = nullptr;         // flipped / transposed fp16 pack for the data gradient
  float* zero_bias = nullptr;
  float* dw_packed = nullptr;        // fp32 [co][k*k][ci] accumulation buffer of the wgmma weight-gradient kernel
  bool dgrad_valid = false;          // w_dgrad matches the current master weights
  int dgrad_n_pad = 0, dgrad_cpad = 0;
};

}  // namespace myolo

using namespace myolo;

struct myolo_plan {
  int B = 0, H = 0, W = 0, num_sms = 132;
  std::vector<myolo_op> ops;
  std::vector<myolo_buf_desc> bufs;
  std::vector<int32_t> extra;
  int32_t* d_extra = nullptr;
  unsigned char* ws = nullptr;
  int64_t ws_bytes = 0;
  std::vector<WeightSlot> slots;
  std::vector<ConvOp> convs;      // parallel to ops (valid for CONV ops)
  std::vector<int> conv_ready;    // tensor maps built
  int64_t last_launches = 0;
  bool force_simt = false;
  // CUDA-graph replay of the internal ops (everything that does not touch caller-owned tensors), captured over several
  // stream "lanes" so that independent branches (C3.cv1 || C3.cv2, seg head || detect head, PSP m8/m16/m32 ...) overlap
  bool warmed = false, use_graph = true, graph_dirty = true;
  std::vector<std::vector<int>> deps;
  std::vector<cudaStream_t> lanes;
  std::vector<cudaEvent_t> op_ev;
  cudaEvent_t ev_start = nullptr;
  cudaEvent_t ev_tail[3] = {nullptr, nullptr, nullptr};   // fork / join of the Detect decodes and the seg upsample behind the graph
  cudaGraph_t graph = nullptr;
  cudaGraphExec_t graph_exec = nullptr;
  int n_graph_ops = 0;
  // training state
  std::vector<BnParams> bns;
  std::vector<float*> bn_stats;       // per op: mean / invstd of the last forward (2*C floats) + 2*C scratch
  unsigned char* gws = nullptr;       // gradient workspace, same layout as ws
  __half* tmp16 = nullptr;            // fp16 copy of an fp32 head gradient / zero-stuffed stride-2 gradient
  size_t tmp16_bytes = 0;
  float* spp_scratch = nullptr;
  size_t spp_scratch_bytes = 0;
  std::vector<ConvOp> dconvs;         // data-gradient convs (parallel to ops)
  std::vector<int> dconv_ready;
  bool train_fwd_done = false;
  // backward replay: one single-lane captured graph per seed mask (bit i = grad_raw[i] given, bit 3 = grad_seg given)
  cudaGraphExec_t bwd_exec[64] = {};   // mask bits 0-2: grad_raw[i], bits 3-5: grad_seg[k] (main / aux16 / aux32 of the BiSe head)
  int bwd_ops[64] = {};
  bool bwd_warm[64] = {};
  float* seg_outs[3] = {nullptr, nullptr, nullptr};          // train forward: extra seg outputs (index 1, 2)
  const float* grad_segs[3] = {nullptr, nullptr, nullptr};   // backward: their gradients
  bool bwd_dirty = false;
  // grouped weight repack (myolo_plan_repack_weights): device job table over all slots, rebuilt when a pointer or pack buffer changed
  PackJob* d_pack_jobs = nullptr;
  int n_pack_jobs = 0, n_pack_chunks = 0, pack_jobs_cap = 0;
  bool pack_table_dirty = true;
  cudaStream_t decode_stream = nullptr;   // low-priority side stream of the Detect decodes (myolo_plan_forward)
  // deferred running statistics (myolo_plan_set_defer_running / myolo_plan_apply_running)
  bool defer_running = false;
  RunningJob* d_run_jobs = nullptr;
  int n_run_jobs = 0;
  unsigned long long seed = 0;       // dropout
  unsigned long long* d_step = nullptr;
  std::vector<cudaEvent_t> bwd_ev;   // per-op completion events of the multi-lane captured backward (+4 join events)
  void* ce_scratch = nullptr;      // 16 bytes for the fused seg loss (valid-pixel count, loss sum)
  float* ce_gbuf = nullptr;        // per-pixel (softmax - onehot), NHWC fp32, of the fused seg loss
  size_t ce_gbuf_bytes = 0;
};

static int resolve_view(const myolo_plan* pl, const myolo_view& v, TensorView* out) {
  MYOLO_REQUIRE(v.buf >= 0 && v.buf < (int)pl->bufs.size(), "view: buffer index %d out of range", v.buf);
  const myolo_buf_desc& bd = pl->bufs[v.buf];
  MYOLO_REQUIRE(v.c_off >= 0 && v.c > 0 && v.c_off + v.c <= bd.c, "view: channel slice [%d,+%d) outside buffer %d (c=%d)", v.c_off,
                v.c, v.buf, bd.c);
  out->dtype = bd.dtype;
  const size_t es = bd.dtype == MYOLO_F16 ? 2 : 4;
  out->base = pl->ws + bd.offset + (size_t)v.c_off * es;
  out->B = pl->B;
  out->H = bd.h;
  out->W = bd.w;
  out->C = v.c;
  out->ctot = bd.c;
  return 0;
}

extern "C" int myolo_abi_version(void) { return MYOLO_ABI_VERSION; }
extern "C" const char* myolo_last_error(void) { return g_err; }

extern "C" int myolo_device_info(char* name, int* sm_count, int* cc_major, int* cc_minor) {
  int dev = 0;
  MYOLO_CHECK_CUDA(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  MYOLO_CHECK_CUDA(cudaGetDeviceProperties(&prop, dev));
  if (name) {
    strncpy(name, prop.name, 255);
    name[255] = 0;
  }
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  return 0;
}

extern "C" int myolo_plan_create(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs, const int32_t* extra,
                                 int n_extra, int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, myolo_plan** out) {
  MYOLO_REQUIRE(ops && bufs && out && n_ops > 0 && n_bufs > 0 && B > 0 && H > 0 && W > 0, "plan_create: bad arguments");
  int sms = 0;
  int rc = check_device(&sms);
  if (rc) return rc;
  myolo_plan* pl = new myolo_plan();
  pl->B = B;
  pl->H = H;
  pl->W = W;
  pl->num_sms = sms;
  pl->ops.assign(ops, ops + n_ops);
  pl->bufs.assign(bufs, bufs + n_bufs);
  if (n_extra > 0) pl->extra.assign(extra, extra + n_extra);
  pl->slots.resize(n_weight_slots);
  pl->convs.resize(n_ops);
  pl->conv_ready.assign(n_ops, 0);
  const char* fs = getenv("MYOLO_FORCE_SIMT");
  pl->force_simt = fs && fs[0] == '1';
  const char* ng = getenv("MYOLO_NO_GRAPH");
  pl->use_graph = !(ng && ng[0] == '1');
  for (int i = 0; i < n_bufs; ++i) {
    const myolo_buf_desc& bd = bufs[i];
    const int64_t bytes = (int64_t)B * bd.h * bd.w * bd.c * (bd.dtype == MYOLO_F16 ? 2 : 4);
    if (bd.offset < 0 || bd.offset % 256 != 0 || bd.offset + bytes > workspace_bytes) {
      set_error("plan_create: buffer %d (offset %lld, %lld bytes) outside workspace of %lld bytes", i, (long long)bd.offset,
                (long long)bytes, (long long)workspace_bytes);
      delete pl;
      return MYOLO_E_INVALID;
    }
  }
  cudaError_t e = cudaMalloc(&pl->ws, workspace_bytes);
  if (e == cudaSuccess) e = cudaMemset(pl->ws, 0, workspace_bytes);
  if (e == cudaSuccess && n_extra > 0) {
    e = cudaMalloc(&pl->d_extra, (size_t)n_extra * 4);
    if (e == cudaSuccess) e = cudaMemcpy(pl->d_extra, extra, (size_t)n_extra * 4, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    set_error("plan_create: device allocation failed: %s", cudaGetErrorString(e));
    if (pl->ws) cudaFree(pl->ws);
    if (pl->d_extra) cudaFree(pl->d_extra);
    delete pl;
    return MYOLO_E_CUDA;
  }
  pl->ws_bytes = workspace_bytes;
  *out = pl;
  return 0;
}

extern "C" void myolo_plan_destroy(myolo_plan* pl) {
  if (!pl) return;
  for (auto& s : pl->slots) {
    if (s.w) cudaFree(s.w);
    if (s.bias) cudaFree(s.bias);
  }
  if (pl->ws) cudaFree(pl->ws);
  if (pl->d_extra) cudaFree(pl->d_extra);
  if (pl->decode_stream) cudaStreamDestroy(pl->decode_stream);
  if (pl->d_pack_jobs) cudaFree(pl->d_pack_jobs);
  if (pl->d_run_jobs) cudaFree(pl->d_run_jobs);
  if (pl->graph_exec) cudaGraphExecDestroy(pl->graph_exec);
  for (auto& e : pl->bwd_exec) if (e) cudaGraphExecDestroy(e);
  if (pl->graph) cudaGraphDestroy(pl->graph);
  for (auto e : pl->op_ev) cudaEventDestroy(e);
  if (pl->ev_start) cudaEventDestroy(pl->ev_start);
  for (auto& e : pl->ev_tail) if (e) cudaEventDestroy(e);
  for (auto st : pl->lanes) cudaStreamDestroy(st);
  for (auto& sl : pl->slots) {
    if (sl.w_dgrad) cudaFree(sl.w_dgrad);
    if (sl.zero_bias) cudaFree(sl.zero_bias);
  }
  for (auto p : pl->bn_stats) if (p) cudaFree(p);
  if (pl->gws) cudaFree(pl->gws);
  for (auto& sl : pl->slots) if (sl.dw_packed) cudaFree(sl.dw_packed);
  if (pl->tmp16) cudaFree(pl->tmp16);
  for (auto e : pl->bwd_ev) cudaEventDestroy(e);
  if (pl->ce_scratch) cudaFree(pl->ce_scratch);
  if (pl->d_step) cudaFree(pl->d_step);
  if (pl->ce_gbuf) cudaFree(pl->ce_gbuf);
  if (pl->spp_scratch) cudaFree(pl->spp_scratch);
  delete pl;
}

static int conv_n_pad(int co) {
  // Co_pad must cover n_tiles_n * BN of the wgmma kernel (see conv_tc_prepare) and stay a multiple of 16 for the simt kernel
  const int co16 = (int)align_up(co, 16);
  if (co16 <= 128) return co16;
  for (int bn = 128; bn >= 16; bn -= 16)
    if (co16 % bn == 0) return co16;
  return co16;
}

extern "C" int myolo_plan_set_conv_weights(myolo_plan* pl, int slot, const float* w, int co, int ci, int k, const float* gamma,
                                           const float* beta, const float* mean, const float* var, float eps, const float* bias,
                                           void* stream) {
  MYOLO_REQUIRE(pl && w && slot >= 0 && slot < (int)pl->slots.size(), "set_conv_weights: bad slot %d", slot);
  MYOLO_REQUIRE((gamma && beta && mean && var) || (!gamma && !beta && !mean && !var), "set_conv_weights: partial BN parameters");
  WeightSlot& s = pl->slots[slot];
  const int co_pad = conv_n_pad(co), ci_pad = (int)align_up(ci, 16);
  if (!s.w || s.co_pad != co_pad || s.ci_pad != ci_pad || s.k != k) {
    if (s.w) cudaFree(s.w);
    if (s.bias) cudaFree(s.bias);
    s.w = nullptr;
    s.bias = nullptr;
    MYOLO_CHECK_CUDA(cudaMalloc(&s.w, (size_t)co_pad * k * k * ci_pad * 2));
    MYOLO_CHECK_CUDA(cudaMalloc(&s.bias, (size_t)co_pad * 4));
    pl->pack_table_dirty = true;
    for (size_t i = 0; i < pl->ops.size(); ++i)
      if (pl->ops[i].kind == MYOLO_OP_CONV && pl->ops[i].weight_slot == slot) pl->conv_ready[i] = 0;
    pl->graph_dirty = true;
  }
  s.co = co;
  s.ci = ci;
  s.k = k;
  s.co_pad = co_pad;
  s.ci_pad = ci_pad;
  s.set = true;
  if (s.w_master != w || s.gamma != gamma || s.beta != beta || s.mean != mean || s.var != var || s.bias_master != bias || s.eps != eps)
    pl->pack_table_dirty = true;
  s.w_master = w;
  s.gamma = gamma;
  s.beta = beta;
  s.mean = mean;
  s.var = var;
  s.bias_master = bias;
  s.eps = eps;
  s.dgrad_valid = false;
  return pack_conv_weights(w, co, ci, k, gamma, beta, mean, var, eps, bias, s.w, s.bias, co_pad, ci_pad, (cudaStream_t)stream);
}

// reference train.py:396-398 changes every parameter once per step; the fp16 copies (forward packs and, once a backward has run, the
// flipped / transposed data-gradient packs) follow in ONE launch from the pointers myolo_plan_set_conv_weights registered
extern "C" int myolo_plan_repack_weights(myolo_plan* pl, void* stream) {
  NvtxRange nvtx("myolo_plan_repack_weights");
  MYOLO_REQUIRE(pl, "repack_weights: null plan");
  cudaStream_t s = (cudaStream_t)stream;
  if (pl->pack_table_dirty) {
    std::vector<PackJob> jobs;
    int chunk = 0;
    for (size_t i = 0; i < pl->slots.size(); ++i) {
      const WeightSlot& sl = pl->slots[i];
      MYOLO_REQUIRE(sl.set && sl.w_master, "repack_weights: slot %d was never set (call myolo_plan_set_conv_weights first)", (int)i);
      PackJob j{sl.w_master, sl.gamma, sl.beta, sl.mean, sl.var, sl.bias_master, sl.w, sl.bias, sl.co, sl.ci, sl.k, sl.co_pad, sl.ci_pad, sl.eps, 0, chunk};
      chunk += (int)(((long)sl.co_pad * sl.k * sl.k * sl.ci_pad + kPackChunk - 1) / kPackChunk);
      jobs.push_back(j);
      if (sl.w_dgrad && sl.dgrad_n_pad > 0) {
        PackJob d{sl.w_master, nullptr, nullptr, nullptr, nullptr, nullptr, sl.w_dgrad, sl.zero_bias, sl.co, sl.ci, sl.k, sl.dgrad_n_pad, sl.dgrad_cpad, 0.f, 1, chunk};
        chunk += (int)(((long)sl.dgrad_n_pad * sl.k * sl.k * sl.dgrad_cpad + kPackChunk - 1) / kPackChunk);
        jobs.push_back(d);
      }
    }
    if ((int)jobs.size() > pl->pack_jobs_cap) {
      if (pl->d_pack_jobs) cudaFree(pl->d_pack_jobs);
      pl->d_pack_jobs = nullptr;
      pl->pack_jobs_cap = (int)jobs.size() + 64;
      MYOLO_CHECK_CUDA(cudaMalloc(&pl->d_pack_jobs, (size_t)pl->pack_jobs_cap * sizeof(PackJob)));
    }
    // rare (first step / first backward / moved parameters): ordered behind the stream's earlier launches of the old table, host-synchronous
    MYOLO_CHECK_CUDA(cudaStreamSynchronize(s));
    MYOLO_CHECK_CUDA(cudaMemcpy(pl->d_pack_jobs, jobs.data(), jobs.size() * sizeof(PackJob), cudaMemcpyHostToDevice));
    pl->n_pack_jobs = (int)jobs.size();
    pl->n_pack_chunks = chunk;
    pl->pack_table_dirty = false;
  }
  int rc = pack_group_launch(pl->d_pack_jobs, pl->n_pack_jobs, pl->n_pack_chunks, s);
  if (rc) return rc;
  g_launch_count++;
  for (auto& sl : pl->slots)
    if (sl.w_dgrad && sl.dgrad_n_pad > 0) sl.dgrad_valid = true;
  return 0;
}

static int prepare_conv(myolo_plan* pl, int i) {
  const myolo_op& op = pl->ops[i];
  MYOLO_REQUIRE(op.weight_slot >= 0 && op.weight_slot < (int)pl->slots.size(), "op %d: bad weight slot", i);
  const WeightSlot& s = pl->slots[op.weight_slot];
  if (!s.set) {
    set_error("op %d: weights of slot %d were never set (call myolo_plan_set_conv_weights first)", i, op.weight_slot);
    return MYOLO_E_STATE;
  }
  ConvOp& c = pl->convs[i];
  c = ConvOp();
  int rc;
  if ((rc = resolve_view(pl, op.in, &c.in))) return rc;
  if ((rc = resolve_view(pl, op.out, &c.out))) return rc;
  c.has_res = op.in2.buf >= 0;
  if (c.has_res && (rc = resolve_view(pl, op.in2, &c.res))) return rc;
  c.k = op.k;
  c.stride = op.stride;
  c.dil = op.dil;
  c.act = op.act;
  c.w = s.w;
  c.bias = s.bias;
  c.Ci_pad = s.ci_pad;
  c.Co_pad = s.co_pad;
  c.Co = s.co;
  MYOLO_REQUIRE(s.k == op.k, "op %d: kernel size %d != packed weights %d", i, op.k, s.k);
  MYOLO_REQUIRE(c.in.C == s.ci_pad, "op %d: input view has %d channels, packed weights expect %d", i, c.in.C, s.ci_pad);
  MYOLO_REQUIRE(c.out.dtype == MYOLO_F32 || c.out.C == s.co, "op %d: output view has %d channels, weights produce %d", i, c.out.C, s.co);
  const int pad = op.dil * (op.k / 2);
  const int ho = (c.in.H + 2 * pad - op.dil * (op.k - 1) - 1) / op.stride + 1;
  const int wo = (c.in.W + 2 * pad - op.dil * (op.k - 1) - 1) / op.stride + 1;
  MYOLO_REQUIRE(ho == c.out.H && wo == c.out.W, "op %d: conv output %dx%d does not match buffer %dx%d", i, ho, wo, c.out.H, c.out.W);
  c.use_tc = !pl->force_simt && !(op.flags & MYOLO_CONV_FORCE_SIMT) && conv_tc_eligible(c);
  if (c.use_tc && (rc = conv_tc_prepare(c, pl->num_sms))) return rc;
  pl->conv_ready[i] = 1;
  return 0;
}

static int run_op(myolo_plan* pl, int i, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                  int64_t* seg_argmax, cudaStream_t s) {
  const myolo_op& op = pl->ops[i];
  TensorView in, in2, out;
  int rc;
  // grouped launches: a run of consecutive ops of one kind executed by the head's launch (include/myolo.h MYOLO_OP_GROUP_*)
  if (op.flags & MYOLO_OP_GROUP_MEMBER) return 0;
  if (op.flags & MYOLO_OP_GROUP_HEAD) {
    const int n = op.aux[7];
    MYOLO_REQUIRE(n >= 2 && n <= 4 && i + n <= (int)pl->ops.size(), "op %d: bad group size %d", i, n);
    for (int j = 1; j < n; ++j)
      MYOLO_REQUIRE(pl->ops[i + j].kind == op.kind && (pl->ops[i + j].flags & MYOLO_OP_GROUP_MEMBER), "op %d: group member %d malformed", i, j);
    if (op.kind == MYOLO_OP_REGION_COMBINE) {
      TensorView outs[4];
      const int* bins[4];
      int nb[4];
      if ((rc = resolve_view(pl, op.in, &in))) return rc;
      for (int j = 0; j < n; ++j) {
        const myolo_op& o = pl->ops[i + j];
        MYOLO_REQUIRE(o.in.buf == op.in.buf && o.aux[2] == op.aux[2], "op %d: grouped region_combine ops must share the atom grid", i + j);
        if ((rc = resolve_view(pl, o.out, &outs[j]))) return rc;
        bins[j] = pl->d_extra + o.aux[0];
        nb[j] = o.aux[1];
      }
      return launch_region_combine_group(in, op.aux[2], bins, nb, outs, n, s);
    }
    if (op.kind == MYOLO_OP_BILINEAR) {
      TensorView ins[4], outs[4];
      for (int j = 0; j < n; ++j)
        if ((rc = resolve_view(pl, pl->ops[i + j].in, &ins[j])) || (rc = resolve_view(pl, pl->ops[i + j].out, &outs[j]))) return rc;
      return launch_bilinear_nhwc_group(ins, outs, n, s);
    }
    if (op.kind == MYOLO_OP_CONV) {
      const ConvOp* cs[4];
      for (int j = 0; j < n; ++j) {
        if (!pl->conv_ready[i + j] && (rc = prepare_conv(pl, i + j))) return rc;
        MYOLO_REQUIRE(!pl->convs[i + j].use_tc, "op %d: only CUDA-core convs can be grouped", i + j);
        cs[j] = &pl->convs[i + j];
      }
      return conv_simt_launch_group(cs, n, s);
    }
    set_error("op %d: kind %d cannot head a group", i, op.kind);
    return MYOLO_E_INVALID;
  }
  switch (op.kind) {
    case MYOLO_OP_INPUT_FOCUS:
      if ((rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_input_focus(x, x_dtype, pl->B, pl->H, pl->W, out, s);
    case MYOLO_OP_FOCUS_CONV: {
      if ((rc = resolve_view(pl, op.out, &out))) return rc;
      MYOLO_REQUIRE(op.weight_slot >= 0 && op.weight_slot < (int)pl->slots.size() && pl->slots[op.weight_slot].set,
                    "op %d: focus_conv weights not set", i);
      const WeightSlot& ws = pl->slots[op.weight_slot];
      MYOLO_REQUIRE(ws.k == 3 && ws.ci == 12 && ws.ci_pad == 16, "op %d: focus_conv expects a 3x3 conv over 12 channels", i);
      return launch_focus_conv(x, x_dtype, pl->B, pl->H, pl->W, ws.w, ws.bias, ws.co, out, s);
    }
    case MYOLO_OP_CONV:
      if (!pl->conv_ready[i] && (rc = prepare_conv(pl, i))) return rc;
      return pl->convs[i].use_tc ? conv_tc_launch(pl->convs[i], s) : conv_simt_launch(pl->convs[i], s);
    case MYOLO_OP_UPSAMPLE_NEAREST:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_upsample_nearest2x(in, out, s);
    case MYOLO_OP_SPP_POOL:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      MYOLO_REQUIRE(op.aux[0] == 3 && op.aux[1] == 5, "spp_pool: only the (5,9,13) pyramid is supported");
      return launch_spp_pool(in, out, op.aux[0], s);
    case MYOLO_OP_BILINEAR:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_bilinear_nhwc(in, out, s);
    case MYOLO_OP_REGION_SUM:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_region_sum(in, pl->d_extra + op.aux[0], op.aux[1], pl->d_extra + op.aux[2], op.aux[3], out, s);
    case MYOLO_OP_REGION_COMBINE:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_region_combine(in, op.aux[2], pl->d_extra + op.aux[0], op.aux[1], out, s);
    case MYOLO_OP_CHANNEL_SCALE:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.in2, &in2))) return rc;
      return launch_channel_scale(in, in2, s);
    case MYOLO_OP_ADD:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.in2, &in2)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_add(in, in2, out, s);
    case MYOLO_OP_BROADCAST:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_broadcast(in, out, s);
    case MYOLO_OP_BN_ACT: {
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      const bool has_res = op.in2.buf >= 0;
      if (has_res && (rc = resolve_view(pl, op.in2, &in2))) return rc;
      MYOLO_REQUIRE(op.aux[0] >= 0 && op.aux[0] < (int)pl->bns.size() && pl->bns[op.aux[0]].set, "op %d: BN slot %d not set", i, op.aux[0]);
      const BnParams& bn = pl->bns[op.aux[0]];
      if ((int)pl->bn_stats.size() <= i) pl->bn_stats.resize(pl->ops.size(), nullptr);
      if (!pl->bn_stats[i]) {     // [mean, invstd | sums (kept zero between launches) | final sums of the backward | ticket]
        MYOLO_CHECK_CUDA(cudaMalloc(&pl->bn_stats[i], (6 * (size_t)bn.C + 4) * sizeof(float)));
        MYOLO_CHECK_CUDA(cudaMemsetAsync(pl->bn_stats[i], 0, (6 * (size_t)bn.C + 4) * sizeof(float), s));
      }
      if ((rc = launch_bn_stats(in, bn, pl->bn_stats[i], pl->bn_stats[i] + 2 * bn.C, s, pl->defer_running))) return rc;
      return launch_bn_act_fwd(in, has_res ? &in2 : nullptr, out, bn, pl->bn_stats[i], op.act, s);
    }
    case MYOLO_OP_ACT:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_act_fwd(in, out, op.act, s);
    case MYOLO_OP_DROPOUT:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      MYOLO_REQUIRE(pl->d_step, "op %d: dropout outside a train forward", i);
      return launch_dropout(in, out, op.faux[0], pl->seed, pl->d_step, (unsigned)op.aux[0], 0, s);
    case MYOLO_OP_CHANNEL_SCALE_OOP:
      if ((rc = resolve_view(pl, op.in, &in)) || (rc = resolve_view(pl, op.in2, &in2)) || (rc = resolve_view(pl, op.out, &out))) return rc;
      return launch_channel_scale_oop(in, in2, out, s);
    case MYOLO_OP_DETECT_DECODE: {
      if ((rc = resolve_view(pl, op.in, &in))) return rc;
      const int level = op.aux[0];
      MYOLO_REQUIRE(z != nullptr || raw != nullptr, "detect_decode: no output pointer");
      return launch_detect_decode(in, op.aux[1], op.aux[2], op.faux[0], reinterpret_cast<const float*>(pl->d_extra + op.aux[5]),
                                  raw ? raw[level] : nullptr, z, op.aux[3], op.aux[4], s);
    }
    case MYOLO_OP_SEG_UPSAMPLE: {
      if ((rc = resolve_view(pl, op.in, &in))) return rc;
      if (op.aux[1] > 0) {     // auxiliary seg outputs of the BiSe head in train mode (reference models/yolo.py:70-79,86): fp32 only
        float* dst = op.aux[1] < 3 ? pl->seg_outs[op.aux[1]] : nullptr;
        return dst ? launch_seg_upsample(in, op.aux[0], pl->H, pl->W, dst, MYOLO_F32, nullptr, s) : 0;
      }
      if (!seg && !seg_argmax) return 0;
      return launch_seg_upsample(in, op.aux[0], pl->H, pl->W, seg, seg_dtype, seg_argmax, s);
    }
    default:
      set_error("op %d: unknown kind %d", i, op.kind);
      return MYOLO_E_INVALID;
  }
}

// ------------------------------------------------------------------------------------------------
// dependency analysis + multi-lane graph capture
// ------------------------------------------------------------------------------------------------
static bool is_external_op(int kind) {
  return kind == MYOLO_OP_INPUT_FOCUS || kind == MYOLO_OP_FOCUS_CONV || kind == MYOLO_OP_DETECT_DECODE || kind == MYOLO_OP_SEG_UPSAMPLE;
}

struct Access { int buf, c_lo, c_hi; int64_t lo, hi; bool write; };

static void add_access(const myolo_plan* pl, const myolo_view& v, bool write, std::vector<Access>& out) {
  if (v.buf < 0) return;
  const myolo_buf_desc& bd = pl->bufs[v.buf];
  const int64_t bytes = (int64_t)pl->B * bd.h * bd.w * bd.c * (bd.dtype == MYOLO_F16 ? 2 : 4);
  out.push_back(Access{v.buf, v.c_off, v.c_off + v.c, bd.offset, bd.offset + bytes, write});
}

static void op_accesses(const myolo_plan* pl, const myolo_op& op, std::vector<Access>& acc) {
  acc.clear();
  add_access(pl, op.in, op.kind == MYOLO_OP_CHANNEL_SCALE, acc);   // channel_scale updates `in` in place
  if (op.kind == MYOLO_OP_CHANNEL_SCALE) add_access(pl, op.in, false, acc);
  add_access(pl, op.in2, false, acc);
  add_access(pl, op.out, true, acc);
}

static bool conflicts(const Access& a, const Access& b) {
  if (!(a.write || b.write)) return false;
  if (a.hi <= b.lo || b.hi <= a.lo) return false;              // disjoint bytes
  if (a.buf == b.buf) return a.c_lo < b.c_hi && b.c_lo < a.c_hi;  // same buffer: only overlapping channel slices collide
  return true;                                                  // different buffers sharing workspace bytes (liveness packing)
}

static void compute_deps(myolo_plan* pl) {
  const int n = (int)pl->ops.size();
  pl->deps.assign(n, {});
  std::vector<std::vector<Access>> acc(n);
  for (int i = 0; i < n; ++i) op_accesses(pl, pl->ops[i], acc[i]);
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < i; ++j) {
      bool c = false;
      for (const Access& a : acc[i]) {
        for (const Access& b : acc[j])
          if (conflicts(a, b)) { c = true; break; }
        if (c) break;
      }
      if (c) pl->deps[i].push_back(j);
    }
}

static int build_graph(myolo_plan* pl) {
  const int n = (int)pl->ops.size();
  static int nl_env = -1;
  if (nl_env < 0) {
    const char* e = getenv("MYOLO_LANES");
    nl_env = e ? std::max(4, std::min(16, atoi(e))) : 4;      // >= 4: the captured backward uses lanes 0-3
  }
  // forward graphs: ONE lane by default.  Every conv launch fills the machine, so branch concurrency buys little, while a multi-lane
  // capture makes the graph runtime spread the nodes over many internal streams - every edge becomes a cross-stream dependency and the
  // programmatic-dependent-launch edges between consecutive convs are lost.  MYOLO_FWD_LANES > 1 restores the branch lanes.
  static int fwd_lanes = -1;
  if (fwd_lanes < 0) {
    const char* e = getenv("MYOLO_FWD_LANES");
    fwd_lanes = e ? std::max(1, std::min(nl_env, atoi(e))) : 1;
  }
  const int NL = nl_env;          // streams / events are sized for the backward's lanes
  const int NLF = fwd_lanes;      // lanes this (forward) capture actually uses
  if (pl->deps.empty()) compute_deps(pl);
  if (pl->lanes.empty()) {
    pl->lanes.resize(NL);
    for (auto& st : pl->lanes) MYOLO_CHECK_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    pl->op_ev.resize(n + NL);
    for (auto& e : pl->op_ev) MYOLO_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    MYOLO_CHECK_CUDA(cudaEventCreateWithFlags(&pl->ev_start, cudaEventDisableTiming));
  }
  if (pl->graph_exec) { cudaGraphExecDestroy(pl->graph_exec); pl->graph_exec = nullptr; }
  if (pl->graph) { cudaGraphDestroy(pl->graph); pl->graph = nullptr; }
  std::vector<int> lane_of(n, -1), lane_last(NL, -1);
  std::vector<char> lane_live(NL, 0);
  cudaStream_t origin = pl->lanes[0];
  MYOLO_CHECK_CUDA(cudaStreamBeginCapture(origin, cudaStreamCaptureModeThreadLocal));
  MYOLO_CHECK_CUDA(cudaEventRecord(pl->ev_start, origin));
  lane_live[0] = 1;
  int rc = 0, count = 0;
  for (int i = 0; i < n && !rc; ++i) {
    if (is_external_op(pl->ops[i].kind)) continue;
    // lane choice: continue on the lane of the most recent dependency if that lane has not moved on, else least recently used lane
    int L = -1, latest = -1;
    for (int d : pl->deps[i])
      if (lane_of[d] >= 0 && d > latest) latest = d;
    if (latest >= 0 && lane_last[lane_of[latest]] == latest) L = lane_of[latest];
    if (L < 0) {
      L = 0;
      for (int k = 1; k < NLF; ++k)
        if (lane_last[k] < lane_last[L]) L = k;
    }
    cudaStream_t st = pl->lanes[L];
    if (!lane_live[L]) {
      if (cudaStreamWaitEvent(st, pl->ev_start, 0) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
      lane_live[L] = 1;
    }
    for (int d : pl->deps[i]) {
      if (lane_of[d] < 0 || lane_of[d] == L) continue;   // external op (ordered by the stream) or same lane (stream order)
      if (cudaStreamWaitEvent(st, pl->op_ev[d], 0) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
    }
    if (rc) break;
    rc = run_op(pl, i, nullptr, 0, nullptr, nullptr, nullptr, 0, nullptr, st);
    if (rc) break;
    if (cudaEventRecord(pl->op_ev[i], st) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
    lane_of[i] = L;
    lane_last[L] = i;
    ++count;
  }
  for (int k = 1; k < NL; ++k) {
    if (!lane_live[k]) continue;
    if (cudaEventRecord(pl->op_ev[n + k], pl->lanes[k]) != cudaSuccess || cudaStreamWaitEvent(origin, pl->op_ev[n + k], 0) != cudaSuccess)
      rc = rc ? rc : MYOLO_E_CUDA;
  }
  cudaGraph_t g = nullptr;
  cudaError_t e = cudaStreamEndCapture(origin, &g);
  if (rc || e != cudaSuccess) {
    if (!rc) { set_error("graph capture failed: %s", cudaGetErrorString(e)); rc = MYOLO_E_CUDA; }
    else if (e != cudaSuccess) cudaGetLastError();
    if (g) cudaGraphDestroy(g);
    return rc;
  }
  pl->graph = g;
  MYOLO_CHECK_CUDA(cudaGraphInstantiate(&pl->graph_exec, g, 0));
  pl->n_graph_ops = count;
  pl->graph_dirty = false;
  return 0;
}

extern "C" int myolo_plan_forward(myolo_plan* pl, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                                  int64_t* seg_argmax, void* stream) {
  NvtxRange nvtx_("myolo_plan_forward");
  MYOLO_REQUIRE(pl && x, "plan_forward: null plan / input");
  cudaStream_t s = (cudaStream_t)stream;
  const int64_t l0 = g_launch_count;
  if (!pl->warmed || !pl->use_graph) {
    // first call (lazy tensor-map / attribute setup happens here) or graphs disabled: plain in-order replay
    for (size_t i = 0; i < pl->ops.size(); ++i) {
      int rc = run_op(pl, (int)i, x, x_dtype, z, raw, seg, seg_dtype, seg_argmax, s);
      if (rc) return rc;
    }
    pl->warmed = true;
    pl->last_launches = g_launch_count - l0;
    return 0;
  }
  if (pl->graph_dirty || !pl->graph_exec) {
    for (size_t i = 0; i < pl->ops.size(); ++i)   // re-resolve convs whose weights moved (outside capture)
      if (pl->ops[i].kind == MYOLO_OP_CONV && !pl->conv_ready[i]) {
        int rc = prepare_conv(pl, (int)i);
        if (rc) return rc;
      }
    int rc = build_graph(pl);
    if (rc) return rc;
  }
  int n_ext = 0;
  for (size_t i = 0; i < pl->ops.size(); ++i)     // ops reading the caller's input: before the graph
    if (pl->ops[i].kind == MYOLO_OP_INPUT_FOCUS || pl->ops[i].kind == MYOLO_OP_FOCUS_CONV) {
      int rc = run_op(pl, (int)i, x, x_dtype, z, raw, seg, seg_dtype, seg_argmax, s);
      if (rc) return rc;
      ++n_ext;
    }
  MYOLO_CHECK_CUDA(cudaGraphLaunch(pl->graph_exec, s));
  // ops writing caller-owned outputs run after the graph: the three Detect decodes (small grids, ~50 us in a row) go to a side stream and
  // overlap the x8 seg upsample (HBM-bound, ~80 us) on the caller's stream; the caller's stream joins before the call returns its outputs
  const bool fork = (seg || seg_argmax) && (z || raw) && pl->lanes.size() > 1;
  if (fork) {
    if (!pl->ev_tail[0])
      for (auto& e : pl->ev_tail) MYOLO_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    if (!pl->decode_stream) {      // lowest priority: the decodes fill the SMs the seg upsample (the step's tail) leaves free, not the reverse
      int least = 0, greatest = 0;
      MYOLO_CHECK_CUDA(cudaDeviceGetStreamPriorityRange(&least, &greatest));
      MYOLO_CHECK_CUDA(cudaStreamCreateWithPriority(&pl->decode_stream, cudaStreamNonBlocking, least));
      // (measured, CUPTI: a kernel that follows a graph launch in the SAME stream starts ~24 us after the graph's last node, one on another
      // stream waiting for an event behind the graph after ~2 us.  Moving the seg upsample to a side stream as well made both kernels start
      // together and share the HBM bandwidth: the starved decode chain then ended the step later than it does now - not adopted)
    }
    MYOLO_CHECK_CUDA(cudaEventRecord(pl->ev_tail[0], s));
    MYOLO_CHECK_CUDA(cudaStreamWaitEvent(pl->decode_stream, pl->ev_tail[0], 0));
  }
  // the seg upsample first (it is the longest kernel of the tail), then the decodes on the low-priority side stream
  for (int pass = 0; pass < 2; ++pass)
  for (size_t i = 0; i < pl->ops.size(); ++i)
    if (pl->ops[i].kind == (pass == 0 ? MYOLO_OP_SEG_UPSAMPLE : MYOLO_OP_DETECT_DECODE)) {
      cudaStream_t st = (fork && pl->ops[i].kind == MYOLO_OP_DETECT_DECODE) ? pl->decode_stream : s;
      int rc = run_op(pl, (int)i, x, x_dtype, z, raw, seg, seg_dtype, seg_argmax, st);
      if (rc) return rc;
      ++n_ext;
    }
  if (fork) {
    MYOLO_CHECK_CUDA(cudaEventRecord(pl->ev_tail[1], pl->decode_stream));
    MYOLO_CHECK_CUDA(cudaStreamWaitEvent(s, pl->ev_tail[1], 0));
  }
  pl->last_launches = pl->n_graph_ops + n_ext;
  return 0;
}

// keeps the stream busy for `ns` nanoseconds: myolo_plan_profile enqueues every op and event behind it, so that the event-to-event times are
// device times of back-to-back kernels and not the CPU's launch cadence (~10 us per op with six tensor maps in the argument list)
__global__ void profile_blocker_kernel(long long ns) {
  long long t0, t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
  do {
    __nanosleep(2000);
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  } while (t - t0 < ns);
}

extern "C" int myolo_plan_profile(myolo_plan* pl, const void* x, int x_dtype, float* z, float* const* raw, void* seg, int seg_dtype,
                                  int64_t* seg_argmax, float* host_ms_per_op, void* stream) {
  NvtxRange nvtx_("myolo_plan_profile");
  MYOLO_REQUIRE(pl && x && host_ms_per_op, "plan_profile: null argument");
  cudaStream_t s = (cudaStream_t)stream;
  const size_t n = pl->ops.size();
  std::vector<cudaEvent_t> ev(n + 1);
  for (auto& e : ev) MYOLO_CHECK_CUDA(cudaEventCreate(&e));
  profile_blocker_kernel<<<1, 1, 0, s>>>(4000000LL);       // 4 ms: longer than the CPU needs to enqueue ~100 launches + events
  MYOLO_CHECK_CUDA(cudaEventRecord(ev[0], s));
  for (size_t i = 0; i < n; ++i) {
    int rc = run_op(pl, (int)i, x, x_dtype, z, raw, seg, seg_dtype, seg_argmax, s);
    if (rc) return rc;
    MYOLO_CHECK_CUDA(cudaEventRecord(ev[i + 1], s));
  }
  MYOLO_CHECK_CUDA(cudaEventSynchronize(ev[n]));
  for (size_t i = 0; i < n; ++i) MYOLO_CHECK_CUDA(cudaEventElapsedTime(&host_ms_per_op[i], ev[i], ev[i + 1]));
  for (auto& e : ev) cudaEventDestroy(e);
  return 0;
}

extern "C" int64_t myolo_plan_last_launch_count(const myolo_plan* pl) { return pl ? pl->last_launches : 0; }

// which kernel a conv op of the plan takes and how it is tiled (valid after the first forward): info[0..11] =
// {1 wgmma / 0 CUDA-core, grid, dynamic smem bytes, BN, pipeline stages, mode (always 0: one TMA box per tap), weights-stationary (always 0),
//  tiles per accumulator round (always 1), total tiles, n tiles in N, kc, CTAs per SM (always 1)}
extern "C" int myolo_plan_conv_info(myolo_plan* pl, int op_index, int32_t* info) {
  MYOLO_REQUIRE(pl && info && op_index >= 0 && op_index < (int)pl->ops.size(), "conv_info: bad arguments");
  MYOLO_REQUIRE(pl->ops[op_index].kind == MYOLO_OP_CONV, "conv_info: op %d is not a conv", op_index);
  int rc;
  if (!pl->conv_ready[op_index] && (rc = prepare_conv(pl, op_index))) return rc;
  const ConvOp& c = pl->convs[op_index];
  for (int i = 0; i < 12; ++i) info[i] = 0;
  info[0] = c.use_tc ? 1 : 0;
  if (c.use_tc) {
    info[1] = c.grid; info[2] = c.smem; info[3] = c.p.BN; info[4] = c.p.num_stages; info[5] = 0;
    info[6] = 0; info[7] = 1; info[8] = c.p.total_tiles; info[9] = c.p.n_tiles_n; info[10] = c.p.kc;
    info[11] = 1;
  }
  return 0;
}

extern "C" int myolo_plan_read_view(myolo_plan* pl, myolo_view view, float* dst, void* stream) {
  MYOLO_REQUIRE(pl && dst, "read_view: null argument");
  TensorView v;
  int rc = resolve_view(pl, view, &v);
  if (rc) return rc;
  return launch_read_view(v, dst, (cudaStream_t)stream);
}

// debug / parity tests: the same slice of the GRADIENT workspace (valid after a backward call)
extern "C" int myolo_plan_read_grad_view(myolo_plan* pl, myolo_view view, float* dst, void* stream) {
  MYOLO_REQUIRE(pl && dst && pl->gws, "read_grad_view: null argument / no backward has run");
  TensorView v;
  int rc = resolve_view(pl, view, &v);
  if (rc) return rc;
  v.base = pl->gws + (reinterpret_cast<unsigned char*>(v.base) - pl->ws);
  return launch_read_view(v, dst, (cudaStream_t)stream);
}


// ------------------------------------------------------------------------------------------------
// training: forward with batch-statistics BN, backward over the op list in reverse (SURVEY.md section 8 row a13)
// ------------------------------------------------------------------------------------------------
extern "C" int myolo_plan_set_bn(myolo_plan* pl, int bn_slot, int channels, float* gamma, float* beta, float* running_mean,
                                 float* running_var, float* d_gamma, float* d_beta, float momentum, float eps) {
  MYOLO_REQUIRE(pl && bn_slot >= 0 && gamma && beta && channels > 0, "set_bn: bad arguments");
  if ((int)pl->bns.size() <= bn_slot) pl->bns.resize(bn_slot + 1);
  BnParams& b = pl->bns[bn_slot];
  if (b.gamma != gamma || b.beta != beta || b.running_mean != running_mean || b.running_var != running_var || b.d_gamma != d_gamma ||
      b.d_beta != d_beta || b.momentum != momentum || b.eps != eps) {
    pl->graph_dirty = true;      // kernel arguments are baked into the captured graphs
    pl->bwd_dirty = true;
    if (pl->d_run_jobs) { cudaFree(pl->d_run_jobs); pl->d_run_jobs = nullptr; pl->n_run_jobs = 0; }
  }
  b.gamma = gamma; b.beta = beta; b.running_mean = running_mean; b.running_var = running_var;
  b.d_gamma = d_gamma; b.d_beta = d_beta; b.momentum = momentum; b.eps = eps; b.C = channels; b.set = true;
  return 0;
}

// Two train-mode forwards of ONE model may run concurrently on two plans (the det and the seg pass of reference train.py:364-392) if the
// running statistics still move in the reference's order: the second plan defers its updates (its BN kernels leave the batch sums in the
// plan's scratch) and applies them with one launch once the first plan's forward has finished.
extern "C" int myolo_plan_set_defer_running(myolo_plan* pl, int defer) {
  MYOLO_REQUIRE(pl, "set_defer_running: null plan");
  if (pl->defer_running != (defer != 0)) pl->graph_dirty = true;     // baked into the captured BN launches
  pl->defer_running = defer != 0;
  return 0;
}

extern "C" int myolo_plan_apply_running(myolo_plan* pl, void* stream) {
  NvtxRange nvtx("myolo_plan_apply_running");
  MYOLO_REQUIRE(pl && pl->defer_running, "apply_running: the plan does not defer its running statistics");
  cudaStream_t s = (cudaStream_t)stream;
  if (!pl->d_run_jobs) {
    std::vector<RunningJob> jobs;
    for (size_t i = 0; i < pl->ops.size(); ++i) {
      const myolo_op& op = pl->ops[i];
      if (op.kind != MYOLO_OP_BN_ACT) continue;
      MYOLO_REQUIRE(i < pl->bn_stats.size() && pl->bn_stats[i], "apply_running: no train forward has run on this plan yet");
      const BnParams& bn = pl->bns[op.aux[0]];
      if (!bn.running_mean) continue;
      TensorView in;
      int rc = resolve_view(pl, op.in, &in);
      if (rc) return rc;
      jobs.push_back(RunningJob{bn.running_mean, bn.running_var, pl->bn_stats[i] + 4 * (size_t)bn.C, bn.C, (long)in.B * in.H * in.W, bn.momentum});
    }
    MYOLO_CHECK_CUDA(cudaMalloc(&pl->d_run_jobs, std::max<size_t>(1, jobs.size()) * sizeof(RunningJob)));
    MYOLO_CHECK_CUDA(cudaMemcpy(pl->d_run_jobs, jobs.data(), jobs.size() * sizeof(RunningJob), cudaMemcpyHostToDevice));
    pl->n_run_jobs = (int)jobs.size();
  }
  return launch_bn_apply_running(pl->d_run_jobs, pl->n_run_jobs, s);
}

extern "C" int myolo_plan_set_seed(myolo_plan* pl, uint64_t seed) {
  MYOLO_REQUIRE(pl, "set_seed: null plan");
  if (pl->seed != seed) { pl->graph_dirty = true; pl->bwd_dirty = true; }   // the seed is a kernel argument of the captured graphs
  pl->seed = seed;
  return 0;
}

extern "C" int myolo_plan_set_conv_grad(myolo_plan* pl, int slot, float* d_weight, float* d_bias) {
  MYOLO_REQUIRE(pl && slot >= 0 && slot < (int)pl->slots.size(), "set_conv_grad: bad slot %d", slot);
  if (pl->slots[slot].d_w != d_weight || pl->slots[slot].d_bias != d_bias) pl->bwd_dirty = true;
  pl->slots[slot].d_w = d_weight;
  pl->slots[slot].d_bias = d_bias;
  return 0;
}

extern "C" int myolo_plan_train_forward(myolo_plan* pl, const void* x, int x_dtype, float* const* raw, float* seg, void* stream);
extern "C" int myolo_plan_train_forward_multi(myolo_plan* pl, const void* x, int x_dtype, float* const* raw, float* const* seg, void* stream) {
  NvtxRange nvtx_("myolo_plan_train_forward");
  MYOLO_REQUIRE(pl, "train_forward: null plan");
  pl->seg_outs[1] = seg ? seg[1] : nullptr;
  pl->seg_outs[2] = seg ? seg[2] : nullptr;
  return myolo_plan_train_forward(pl, x, x_dtype, raw, seg ? seg[0] : nullptr, stream);
}

extern "C" int myolo_plan_train_forward(myolo_plan* pl, const void* x, int x_dtype, float* const* raw, float* seg, void* stream) {
  MYOLO_REQUIRE(pl && x, "train_forward: null plan / input");
  if (!pl->d_step) {
    MYOLO_CHECK_CUDA(cudaMalloc(&pl->d_step, sizeof(unsigned long long)));
    MYOLO_CHECK_CUDA(cudaMemset(pl->d_step, 0, sizeof(unsigned long long)));
  }
  {   // a new dropout mask per forward; the counter lives on the device so that captured graphs see the new value
    int brc = launch_bump_step(pl->d_step, (cudaStream_t)stream);
    if (brc) return brc;
  }
  // same executor as inference: first call in order (lazy allocations / tensor maps), then multi-lane CUDA-graph replay of the internal
  // ops with the input conversion before and the caller-owned outputs (raw x_i, seg logits) after the graph
  int rc = myolo_plan_forward(pl, x, x_dtype, nullptr, raw, seg, MYOLO_F32, nullptr, stream);
  if (rc) return rc;
  pl->train_fwd_done = true;
  return 0;
}

static int grad_view(const myolo_plan* pl, const myolo_view& v, TensorView* out) {
  int rc = resolve_view(pl, v, out);
  if (rc) return rc;
  out->base = pl->gws + (reinterpret_cast<unsigned char*>(out->base) - pl->ws);   // same layout in the gradient workspace
  return 0;
}

static int ensure_scratch(myolo_plan* pl, size_t bytes) {      // fp32 scratch shared by the pooling / resampling adjoints (stream ordered)
  if (pl->spp_scratch_bytes >= bytes) return 0;
  if (pl->spp_scratch) cudaFree(pl->spp_scratch);
  pl->spp_scratch = nullptr;
  pl->spp_scratch_bytes = 0;
  MYOLO_CHECK_CUDA(cudaMalloc(&pl->spp_scratch, bytes));
  pl->spp_scratch_bytes = bytes;
  pl->bwd_dirty = true;
  return 0;
}

static int ensure_tmp16(myolo_plan* pl, size_t bytes) {
  if (pl->tmp16_bytes >= bytes) return 0;
  if (pl->tmp16) cudaFree(pl->tmp16);
  pl->tmp16 = nullptr;
  MYOLO_CHECK_CUDA(cudaMalloc(&pl->tmp16, bytes));
  pl->tmp16_bytes = bytes;
  for (auto& r : pl->dconv_ready) r = 0;   // tensor maps point into tmp16
  pl->bwd_dirty = true;
  return 0;
}

// backward of one conv op: dY = grad(out); grad(in) += conv^T(dY, W); dW += ...; dbias += ...
// `ws`: stream of the weight / bias gradient kernels.  Nothing downstream in the backward pass reads them, so the walk forks them onto a
// side lane (ws != s) where they overlap the latency-bound chain of data-gradient / BN kernels; the caller joins the lane at the end.
static int conv_backward(myolo_plan* pl, int i, bool need_dgrad, cudaStream_t s, cudaStream_t ws, bool* used_side) {
  const myolo_op& op = pl->ops[i];
  WeightSlot& sl = pl->slots[op.weight_slot];
  MYOLO_REQUIRE(sl.set && sl.w_master && sl.d_w, "op %d: conv slot %d has no master weights / gradient pointer", i, op.weight_slot);
  TensorView xin, gout, gin;
  int rc;
  if ((rc = resolve_view(pl, op.in, &xin)) || (rc = grad_view(pl, op.out, &gout)) || (rc = grad_view(pl, op.in, &gin))) return rc;
  const long npix_out = (long)gout.B * gout.H * gout.W;
  // tiny maps / fp32 inputs: generic kernels on the fp32 master weights
  if (xin.dtype == MYOLO_F32 || npix_out <= 1024 || gout.H * gout.W < 128) {
    TensorView gy = gout;
    gy.C = sl.co;
    return launch_conv_small_bwd(xin, gy, need_dgrad ? &gin : nullptr, sl.w_master, sl.d_w, sl.d_bias, sl.co, sl.ci, op.k, op.stride, op.dil, s);
  }
  // dY in fp16 (cast fp32 head gradients; zero-stuff for stride 2)
  const int cpad = (int)align_up(sl.co, 16);
  TensorView dy16 = gout;
  size_t need = 0;
  if (gout.dtype == MYOLO_F32) need = (size_t)npix_out * cpad * 2;
  const bool s2 = op.stride == 2;
  size_t stuffed_off = align_up((int64_t)need, 256);
  if (s2) need = stuffed_off + (size_t)gout.B * (2 * gout.H) * (2 * gout.W) * cpad * 2;
  if (need && (rc = ensure_tmp16(pl, need))) return rc;
  if (gout.dtype == MYOLO_F32) {
    dy16 = TensorView{pl->tmp16, gout.B, gout.H, gout.W, cpad, cpad, MYOLO_F16};
    if ((rc = launch_cast_f32_to_f16(gout, dy16, s))) return rc;
  } else {
    MYOLO_REQUIRE(gout.C == sl.co && sl.co % 16 == 0, "op %d: fp16 conv gradient needs Co %% 16 == 0 (Co=%d)", i, sl.co);
  }
  // weight / bias gradients
  // dY in the shared fp16 scratch (fp32 head gradients) is overwritten by the next conv: those few layers stay on the main stream
  cudaStream_t wst = (ws != s && gout.dtype != MYOLO_F32 && (int)pl->op_ev.size() > i) ? ws : s;
  if (wst != s) {
    MYOLO_CHECK_CUDA(cudaEventRecord(pl->op_ev[i], s));          // dY (and everything before it on the main chain) is final here
    MYOLO_CHECK_CUDA(cudaStreamWaitEvent(wst, pl->op_ev[i], 0));
    *used_side = true;
  }
  if (conv_wgrad_tc_eligible(xin, dy16, op.k, op.stride, op.dil, sl.co, sl.ci)) {
    const size_t nb = conv_wgrad_packed_bytes(sl.d_w, sl.co, sl.ci, op.k);
    if (!sl.dw_packed && nb) {
      MYOLO_CHECK_CUDA(cudaMalloc(&sl.dw_packed, nb));
      MYOLO_CHECK_CUDA(cudaMemset(sl.dw_packed, 0, nb));
    }
    if ((rc = launch_conv_wgrad_tc(xin, dy16, op.k, op.stride, op.dil, sl.d_w, sl.dw_packed, sl.co, sl.ci, pl->num_sms, wst))) return rc;
  } else if ((rc = launch_conv_wgrad(xin, dy16, op.k, op.stride, op.dil, sl.d_w, sl.co, sl.ci, nullptr, wst))) {
    return rc;
  }
  if (sl.d_bias) {   // the bias gradient of an fp32 head gradient is summed from the fp32 values, not from their fp16 cast
    TensorView gy = gout.dtype == MYOLO_F32 ? gout : dy16;
    gy.C = sl.co;
    if ((rc = launch_bias_grad(gy, sl.d_bias, sl.co, wst))) return rc;
  }
  if (!need_dgrad) return 0;
  // data gradient = stride-1 conv of (zero-stuffed) dY with flipped / transposed weights, accumulated into grad(in)
  const int ci_out_pad = (int)align_up(sl.ci, 16);
  const int n_pad = ((ci_out_pad <= 128) ? ci_out_pad : [&] { for (int bn = 128; bn >= 16; bn -= 16) if (ci_out_pad % bn == 0) return ci_out_pad; return ci_out_pad; }());
  if (!sl.w_dgrad) {
    MYOLO_CHECK_CUDA(cudaMalloc(&sl.w_dgrad, (size_t)n_pad * op.k * op.k * cpad * 2));
    MYOLO_CHECK_CUDA(cudaMalloc(&sl.zero_bias, (size_t)n_pad * 4));
    pl->pack_table_dirty = true;
  }
  if (!sl.dgrad_valid) {   // (first use; later refreshes happen in refresh_dgrad_packs, outside any captured graph)
    if ((rc = pack_dgrad_weights(sl.w_master, sl.co, sl.ci, op.k, sl.w_dgrad, sl.zero_bias, n_pad, cpad, s))) return rc;
    sl.dgrad_valid = true;
    sl.dgrad_n_pad = n_pad;
    sl.dgrad_cpad = cpad;
  }
  TensorView din = dy16;
  if (s2) {
    din = TensorView{reinterpret_cast<unsigned char*>(pl->tmp16) + stuffed_off, gout.B, 2 * gout.H, 2 * gout.W, cpad, cpad, MYOLO_F16};
    TensorView src = dy16;
    src.C = cpad;
    if (gout.dtype != MYOLO_F32) { src = gout; }
    MYOLO_REQUIRE(src.C == cpad, "op %d: stride-2 gradient channel padding mismatch", i);
    if ((rc = launch_zero_stuff2(src, din, s))) return rc;
  }
  if (pl->dconvs.size() != pl->ops.size()) { pl->dconvs.resize(pl->ops.size()); pl->dconv_ready.assign(pl->ops.size(), 0); }
  ConvOp& c = pl->dconvs[i];
  if (!pl->dconv_ready[i]) {
    c = ConvOp();
    c.in = din;
    c.in.C = cpad;
    c.out = gin;
    c.out.C = sl.ci;
    c.has_res = true;
    c.res = c.out;
    c.k = op.k;
    c.stride = 1;
    c.dil = op.dil;
    c.act = MYOLO_ACT_NONE;
    c.w = sl.w_dgrad;
    c.bias = sl.zero_bias;
    c.Ci_pad = cpad;
    c.Co_pad = n_pad;
    c.Co = sl.ci;
    MYOLO_REQUIRE(din.H == gin.H && din.W == gin.W, "op %d: data-gradient geometry %dx%d vs %dx%d", i, din.H, din.W, gin.H, gin.W);
    c.use_tc = !pl->force_simt && conv_tc_eligible(c);
    if (c.use_tc && (rc = conv_tc_prepare(c, pl->num_sms))) return rc;
    pl->dconv_ready[i] = 1;
  }
  return c.use_tc ? conv_tc_launch(c, s) : conv_simt_launch(c, s);
}

// seeds: dL/d(raw x_i) and dL/d(seg) written into the gradient buffers of the head convs (caller-owned memory: never captured)
static int backward_seeds(myolo_plan* pl, const float* const* grad_raw, const float* grad_seg, std::vector<char>& live, cudaStream_t s) {
  for (int i = (int)pl->ops.size() - 1; i >= 0; --i) {
    const myolo_op& op = pl->ops[i];
    TensorView a;
    int rc;
    if (op.kind == MYOLO_OP_SEG_UPSAMPLE) {
      const float* g = op.aux[1] == 0 ? grad_seg : (op.aux[1] < 3 ? pl->grad_segs[op.aux[1]] : nullptr);
      if (!g) continue;
      if ((rc = grad_view(pl, op.in, &a))) return rc;
      live[op.in.buf] = 1;
      if ((rc = launch_seg_upsample_bwd(g, op.aux[0], pl->H, pl->W, a, s))) return rc;
    } else if (op.kind == MYOLO_OP_DETECT_DECODE && grad_raw && grad_raw[op.aux[0]]) {
      if ((rc = grad_view(pl, op.in, &a))) return rc;
      live[op.in.buf] = 1;
      if ((rc = launch_detect_raw_bwd(grad_raw[op.aux[0]], op.aux[1], op.aux[2], a, s))) return rc;
    }
  }
  return 0;
}

// data-gradient weight packs follow the master weights; refreshed here (never inside a captured graph)
static int refresh_dgrad_packs(myolo_plan* pl, cudaStream_t s) {
  for (auto& sl : pl->slots)
    if (sl.w_dgrad && !sl.dgrad_valid) {
      int rc = pack_dgrad_weights(sl.w_master, sl.co, sl.ci, sl.k, sl.w_dgrad, sl.zero_bias, sl.dgrad_n_pad, sl.dgrad_cpad, s);
      if (rc) return rc;
      sl.dgrad_valid = true;
    }
  return 0;
}

static int backward_walk(myolo_plan* pl, std::vector<char>& live, cudaStream_t s, int* n_ops);

static int backward_run(myolo_plan* pl, int mask, std::vector<char>& live, cudaStream_t s) {
  int rc;
  if ((rc = refresh_dgrad_packs(pl, s))) return rc;
  if (pl->bwd_dirty) {
    for (auto& e : pl->bwd_exec) if (e) { cudaGraphExecDestroy(e); e = nullptr; }
    for (auto& w : pl->bwd_warm) w = false;
    pl->bwd_dirty = false;
  }
  int n_ops = 0;
  if (!pl->use_graph || !pl->bwd_warm[mask]) {
    // first backward with this seed set: in order on the caller's stream (allocations, tensor maps, weight packs happen here)
    rc = backward_walk(pl, live, s, &n_ops);
    if (!rc && !pl->bwd_dirty) pl->bwd_warm[mask] = true;
    return rc;
  }
  if (!pl->bwd_exec[mask]) {
    if (pl->lanes.empty()) { set_error("backward: forward graph state missing"); return MYOLO_E_INVALID; }
    if (pl->bwd_ev.size() < pl->ops.size() + 4) {
      const size_t old_n = pl->bwd_ev.size();
      pl->bwd_ev.resize(pl->ops.size() + 4);
      for (size_t k = old_n; k < pl->bwd_ev.size(); ++k) MYOLO_CHECK_CUDA(cudaEventCreateWithFlags(&pl->bwd_ev[k], cudaEventDisableTiming));
    }
    cudaStream_t cs = pl->lanes[0];
    MYOLO_CHECK_CUDA(cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    rc = backward_walk(pl, live, cs, &n_ops);
    cudaGraph_t g = nullptr;
    cudaError_t e = cudaStreamEndCapture(cs, &g);
    if (rc || e != cudaSuccess || pl->bwd_dirty) {
      if (!rc && e != cudaSuccess) { set_error("backward graph capture failed: %s", cudaGetErrorString(e)); rc = MYOLO_E_CUDA; }
      if (!rc) { set_error("backward graph capture needed a (re)allocation"); rc = MYOLO_E_INVALID; }
      cudaGetLastError();
      if (g) cudaGraphDestroy(g);
      return rc;
    }
    cudaError_t ie = cudaGraphInstantiate(&pl->bwd_exec[mask], g, 0);
    cudaGraphDestroy(g);
    MYOLO_CHECK_CUDA(ie);
    pl->bwd_ops[mask] = n_ops;
  }
  MYOLO_CHECK_CUDA(cudaGraphLaunch(pl->bwd_exec[mask], s));
  return 0;
}

extern "C" int myolo_plan_backward(myolo_plan* pl, const float* const* grad_raw, const float* grad_seg, void* stream);
extern "C" int myolo_plan_backward_multi(myolo_plan* pl, const float* const* grad_raw, const float* const* grad_seg, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward");
  MYOLO_REQUIRE(pl, "backward: null plan");
  pl->grad_segs[1] = grad_seg ? grad_seg[1] : nullptr;
  pl->grad_segs[2] = grad_seg ? grad_seg[2] : nullptr;
  int rc = myolo_plan_backward(pl, grad_raw, grad_seg ? grad_seg[0] : nullptr, stream);
  pl->grad_segs[1] = pl->grad_segs[2] = nullptr;
  return rc;
}

extern "C" int myolo_plan_backward(myolo_plan* pl, const float* const* grad_raw, const float* grad_seg, void* stream) {
  MYOLO_REQUIRE(pl && pl->train_fwd_done, "backward: call myolo_plan_train_forward first");
  cudaStream_t s = (cudaStream_t)stream;
  if (!pl->gws) MYOLO_CHECK_CUDA(cudaMalloc(&pl->gws, pl->ws_bytes));
  MYOLO_CHECK_CUDA(cudaMemsetAsync(pl->gws, 0, pl->ws_bytes, s));
  int mask = (grad_seg ? 8 : 0) | (pl->grad_segs[1] ? 16 : 0) | (pl->grad_segs[2] ? 32 : 0);
  for (int i = 0; i < 3; ++i)
    if (grad_raw && grad_raw[i]) mask |= 1 << i;
  // Buffers whose gradient is still all-zero are tracked, and ops that would only propagate zeros are skipped: the det pass of an
  // iteration never touches the seg head, the seg pass never the Detect convs (reference train.py:364-392 runs two passes).
  std::vector<char> live(pl->bufs.size(), 0);
  int rc = backward_seeds(pl, grad_raw, grad_seg, live, s);
  if (rc) return rc;
  return backward_run(pl, mask, live, s);
}

// fused seg loss (SURVEY.md section 8f rank 3): CE(ignore_index) of the x8-upsampled logits of the last train forward is evaluated and
// differentiated straight from the low-resolution logits; the backward then runs as the seg pass (seed mask 8)
extern "C" int myolo_plan_backward_seg_ce(myolo_plan* pl, const int64_t* labels, int ignore_index, float factor, const float* scale_dev,
                                          float* loss_out, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward_seg_ce");
  MYOLO_REQUIRE(pl && pl->train_fwd_done && labels, "backward_seg_ce: call myolo_plan_train_forward first / null labels");
  cudaStream_t s = (cudaStream_t)stream;
  if (!pl->gws) MYOLO_CHECK_CUDA(cudaMalloc(&pl->gws, pl->ws_bytes));
  MYOLO_CHECK_CUDA(cudaMemsetAsync(pl->gws, 0, pl->ws_bytes, s));
  if (!pl->ce_scratch) MYOLO_CHECK_CUDA(cudaMalloc(&pl->ce_scratch, 16));
  std::vector<char> live(pl->bufs.size(), 0);
  int rc = MYOLO_E_INVALID;
  for (const auto& op : pl->ops)
    if (op.kind == MYOLO_OP_SEG_UPSAMPLE) {
      TensorView lo, dlo;
      if ((rc = resolve_view(pl, op.in, &lo)) || (rc = grad_view(pl, op.in, &dlo))) return rc;
      live[op.in.buf] = 1;
      const size_t gb = seg_ce_scratch_bytes(pl->B, pl->H, pl->W, op.aux[0]);
      if (pl->ce_gbuf_bytes < gb) {
        if (pl->ce_gbuf) cudaFree(pl->ce_gbuf);
        pl->ce_gbuf = nullptr;
        pl->ce_gbuf_bytes = 0;
        MYOLO_CHECK_CUDA(cudaMalloc(&pl->ce_gbuf, gb));
        pl->ce_gbuf_bytes = gb;
      }
      rc = launch_seg_ce_fused(lo, op.aux[0], reinterpret_cast<const long long*>(labels), pl->H, pl->W, ignore_index, dlo, factor, scale_dev,
                               pl->ce_scratch, pl->ce_gbuf, loss_out, s);
      break;
    }
  if (rc) { if (rc == MYOLO_E_INVALID) set_error("backward_seg_ce: the plan has no segmentation output"); return rc; }
  return backward_run(pl, 8, live, s);
}

static int backward_walk(myolo_plan* pl, std::vector<char>& live, cudaStream_t s, int* n_ops) {
  const int n = (int)pl->ops.size();
  // which buffers are produced by the input conversion (no data gradient needed into them)
  std::vector<char> is_input_buf(pl->bufs.size(), 0);
  for (const auto& op : pl->ops)
    if (op.kind == MYOLO_OP_INPUT_FOCUS && op.out.buf >= 0) is_input_buf[op.out.buf] = 1;
  int rc = 0;
  auto is_live = [&](const myolo_view& v) { return v.buf >= 0 && live[v.buf]; };
  auto mark = [&](const myolo_view& v) { if (v.buf >= 0) live[v.buf] = 1; };
  static int side_env = -1;
  if (side_env < 0) {
    const char* e = getenv("MYOLO_WGRAD_LANE");
    side_env = e ? atoi(e) : 1;
  }
  // weight-gradient lane (exists once the forward graph has created the plan's streams / events)
  cudaStream_t side = (side_env && pl->lanes.size() >= 2 && pl->lanes[1] != s && (int)pl->op_ev.size() >= n + 2) ? pl->lanes[1] : s;
  bool used_side = false;
  // Under capture the chain itself is spread over three lanes: ops are ordered only by real dependencies on the GRADIENT buffers
  // (reads of grad(out), read-modify-writes of grad(in) / grad(in2)) and on the two shared scratch areas, so the branches of C3 /
  // SPP / PSP / the three detect levels overlap exactly as they do in the forward graph.
  static int ml_env = -1;
  if (ml_env < 0) {
    const char* e = getenv("MYOLO_BWD_LANES");
    ml_env = e ? atoi(e) : 0;     // like the forward graph, a multi-lane capture is spread over dozens of internal streams and every edge
                                  // becomes a cross-stream wait
  }
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(s, &cap);
  const bool multi = ml_env && cap == cudaStreamCaptureStatusActive && pl->lanes.size() >= 4 && s == pl->lanes[0] &&
                     (int)pl->bwd_ev.size() >= n + 4;
  struct GAcc { int buf, c_lo, c_hi; bool write; };
  auto acc_of = [&](int i, std::vector<GAcc>& out) {
    const myolo_op& op = pl->ops[i];
    out.clear();
    auto add = [&](const myolo_view& v, bool w) { if (v.buf >= 0) out.push_back(GAcc{v.buf, v.c_off, v.c_off + v.c, w}); };
    add(op.out, false);
    add(op.in, true);
    add(op.in2, true);
    if (op.kind == MYOLO_OP_CONV && (op.stride == 2 || pl->bufs[op.out.buf].dtype == MYOLO_F32)) out.push_back(GAcc{-2, 0, 1, true});  // tmp16
    if (op.kind == MYOLO_OP_BILINEAR || op.kind == MYOLO_OP_SPP_POOL) out.push_back(GAcc{-3, 0, 1, true});                          // fp32 scratch
  };
  std::vector<int> done;                       // executed ops, in execution order
  std::vector<std::vector<GAcc>> done_acc;
  std::vector<int> lane_of(n, -1);
  const int NLc = 3;
  cudaStream_t chain[NLc] = {s, multi ? pl->lanes[2] : s, multi ? pl->lanes[3] : s};
  int lane_last[NLc] = {-1, -1, -1};           // position (in `done`) of the last op of each lane
  bool lane_used[NLc] = {true, false, false};
  if (multi) {
    if (cudaEventRecord(pl->bwd_ev[n], s) != cudaSuccess) { set_error("backward: capture fork failed"); return MYOLO_E_CUDA; }
  }
  std::vector<GAcc> cur;
  for (int i = n - 1; i >= 0 && !rc; --i) {
    const myolo_op& op = pl->ops[i];
    TensorView a, b, c, d;
    if (op.kind == MYOLO_OP_SEG_UPSAMPLE || op.kind == MYOLO_OP_DETECT_DECODE || op.kind == MYOLO_OP_INPUT_FOCUS) continue;
    if (!is_live(op.out)) continue;
    mark(op.in);
    mark(op.in2);
    ++*n_ops;
    cudaStream_t s = chain[0];                 // (shadows the origin: the op's lane)
    int L = 0;
    if (multi) {
      acc_of(i, cur);
      std::vector<int> deps;                   // positions in `done`
      for (int q = (int)done.size() - 1; q >= 0; --q) {
        bool hit = false;
        for (const GAcc& x : cur) {
          for (const GAcc& y : done_acc[q])
            if (x.buf == y.buf && (x.write || y.write) && x.c_lo < y.c_hi && y.c_lo < x.c_hi) { hit = true; break; }
          if (hit) break;
        }
        if (hit) deps.push_back(q);
      }
      int latest = deps.empty() ? -1 : deps.front();         // deps are in decreasing position order
      L = -1;
      if (latest >= 0 && lane_last[lane_of[done[latest]]] == latest) L = lane_of[done[latest]];
      if (L < 0) {
        L = 0;
        for (int k = 1; k < NLc; ++k)
          if (lane_last[k] < lane_last[L]) L = k;
      }
      s = chain[L];
      if (!lane_used[L]) {
        if (cudaStreamWaitEvent(s, pl->bwd_ev[n], 0) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
        lane_used[L] = true;
      }
      for (int q : deps) {
        if (lane_of[done[q]] == L) continue;
        if (cudaStreamWaitEvent(s, pl->bwd_ev[done[q]], 0) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
      }
      if (rc) break;
    }
    switch (op.kind) {
      case MYOLO_OP_CONV:
        rc = conv_backward(pl, i, !is_input_buf[op.in.buf], s, side, &used_side);
        break;
      case MYOLO_OP_BN_ACT: {
        const bool has_res = op.in2.buf >= 0;
        if ((rc = resolve_view(pl, op.in, &a)) || (rc = grad_view(pl, op.out, &b)) || (rc = grad_view(pl, op.in, &c))) break;
        if (has_res && (rc = grad_view(pl, op.in2, &d))) break;
        const BnParams& bn = pl->bns[op.aux[0]];
        rc = launch_bn_act_bwd(a, b, c, has_res ? &d : nullptr, bn, pl->bn_stats[i], op.act, pl->bn_stats[i] + 2 * bn.C, s);
        break;
      }
      case MYOLO_OP_ACT:
        if ((rc = resolve_view(pl, op.in, &a)) || (rc = grad_view(pl, op.out, &b)) || (rc = grad_view(pl, op.in, &c))) break;
        rc = launch_act_bwd(a, b, c, op.act, s);
        break;
      case MYOLO_OP_DROPOUT:
        if ((rc = grad_view(pl, op.out, &b)) || (rc = grad_view(pl, op.in, &c))) break;
        rc = launch_dropout(b, c, op.faux[0], pl->seed, pl->d_step, (unsigned)op.aux[0], 1, s);
        break;
      case MYOLO_OP_ADD:          // out = in + in2: both inputs receive the output gradient
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b)) || (rc = grad_view(pl, op.in2, &c))) break;
        if ((rc = launch_grad_add(a, b, s))) break;
        rc = launch_grad_add(a, c, s);
        break;
      case MYOLO_OP_BROADCAST:    // out[b,y,x,c] = in[b,0,0,c]: the 1x1 map receives the per-image spatial sum
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b))) break;
        rc = launch_broadcast_bwd(a, b, s);
        break;
      case MYOLO_OP_CHANNEL_SCALE_OOP: {
        TensorView f, av, gout, gf, ga;
        if ((rc = resolve_view(pl, op.in, &f)) || (rc = resolve_view(pl, op.in2, &av)) || (rc = grad_view(pl, op.out, &gout)) ||
            (rc = grad_view(pl, op.in, &gf)) || (rc = grad_view(pl, op.in2, &ga)))
          break;
        rc = launch_channel_scale_bwd(f, av, gout, gf, ga, s);
        break;
      }
      case MYOLO_OP_UPSAMPLE_NEAREST:
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b))) break;
        rc = launch_nearest2x_bwd(a, b, s);
        break;
      case MYOLO_OP_BILINEAR:
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b))) break;
        if ((rc = ensure_scratch(pl, bilinear_bwd_scratch_bytes(a, b)))) break;
        rc = launch_bilinear_bwd(a, b, pl->spp_scratch, s);
        break;
      case MYOLO_OP_SPP_POOL: {
        if ((rc = resolve_view(pl, op.in, &a)) || (rc = grad_view(pl, op.out, &b)) || (rc = grad_view(pl, op.in, &c))) break;
        if ((rc = ensure_scratch(pl, (size_t)a.B * a.H * a.W * a.C * sizeof(float)))) break;
        rc = launch_spp_bwd(a, b, c, pl->spp_scratch, s);
        break;
      }
      case MYOLO_OP_REGION_COMBINE:
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b))) break;
        rc = launch_region_combine_bwd(a, b, op.aux[2], pl->d_extra + op.aux[0], op.aux[1], s);
        break;
      case MYOLO_OP_REGION_SUM:
        if ((rc = grad_view(pl, op.out, &a)) || (rc = grad_view(pl, op.in, &b))) break;
        rc = launch_region_bwd(a, b, pl->d_extra + op.aux[0], op.aux[1], pl->d_extra + op.aux[2], op.aux[3], s);
        break;
      default:
        set_error("backward: op %d of kind %d has no backward", i, op.kind);
        rc = MYOLO_E_INVALID;
    }
    if (multi && !rc) {
      if (cudaEventRecord(pl->bwd_ev[i], s) != cudaSuccess) { rc = MYOLO_E_CUDA; break; }
      lane_of[i] = L;
      done.push_back(i);
      done_acc.push_back(cur);
      lane_last[L] = (int)done.size() - 1;
    }
  }
  if (multi) {   // join the chain lanes into the origin
    for (int k = 1; k < NLc; ++k)
      if (lane_used[k] && (cudaEventRecord(pl->bwd_ev[n + k], chain[k]) != cudaSuccess || cudaStreamWaitEvent(chain[0], pl->bwd_ev[n + k], 0) != cudaSuccess))
        if (!rc) { set_error("backward: joining the capture lanes failed"); rc = MYOLO_E_CUDA; }
  }
  if (used_side) {   // join the weight-gradient lane (required to close a capture; in eager mode it orders the optimiser after it)
    if (cudaEventRecord(pl->op_ev[n + 1], side) != cudaSuccess || cudaStreamWaitEvent(s, pl->op_ev[n + 1], 0) != cudaSuccess) {
      if (!rc) { set_error("backward: joining the weight-gradient lane failed"); rc = MYOLO_E_CUDA; }
    }
  }
  return rc;
}

extern "C" int myolo_letterbox(const uint8_t* src, int B, int H0, int W0, int resized_w, int resized_h, int top, int left, int H, int W,
                               const int32_t* pad_bgr, void* out, int out_dtype, int chw, int swap_rb, void* stream) {
  int rc = check_device(nullptr);
  if (rc) return rc;
  return launch_letterbox(src, B, H0, W0, resized_w, resized_h, top, left, H, W, pad_bgr, out, out_dtype, chw, swap_rb, (cudaStream_t)stream);
}

extern "C" int myolo_seg_lut_blend(const void* class_map, int map_dtype, int64_t n_pixels, const uint8_t* lut, int n_entries, int channels,
                                   int reverse_channels, uint8_t* out, const uint8_t* image, float alpha, float beta, uint8_t* blend,
                                   void* stream) {
  int rc = check_device(nullptr);
  if (rc) return rc;
  return launch_lut_blend(class_map, map_dtype, (long)n_pixels, lut, n_entries, channels, reverse_channels, out, image, alpha, beta, blend,
                          (cudaStream_t)stream);
}

extern "C" int myolo_seg_metrics(const void* pred, int pred_dtype, const int64_t* target, int64_t n_pixels, int n_classes, uint64_t* counters,
                                 void* stream) {
  int rc = check_device(nullptr);
  if (rc) return rc;
  return launch_seg_hist(pred, pred_dtype, reinterpret_cast<const long long*>(target), (long)n_pixels, n_classes,
                         reinterpret_cast<unsigned long long*>(counters), (cudaStream_t)stream);
}

extern "C" int myolo_conv_wgrad(const void* x, const void* dy, int B, int H, int W, int ci, int co, int k, int stride, int dil, float* dW,
                                int path, void* stream) {
  MYOLO_REQUIRE(x && dy && dW && B > 0 && (k == 1 || k == 3) && (stride == 1 || stride == 2), "conv_wgrad: bad arguments");
  int sms = 0;
  int rc = check_device(&sms);
  if (rc) return rc;
  const int pad = dil * (k / 2);
  const int Ho = (H + 2 * pad - dil * (k - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  TensorView xv{const_cast<void*>(x), B, H, W, ci, ci, MYOLO_F16};
  TensorView dv{const_cast<void*>(dy), B, Ho, Wo, co, co, MYOLO_F16};
  cudaStream_t s = (cudaStream_t)stream;
  if (path == 0) return launch_conv_wgrad(xv, dv, k, stride, dil, dW, co, ci, nullptr, s);
  MYOLO_REQUIRE(conv_wgrad_tc_eligible(xv, dv, k, stride, dil, co, ci), "conv_wgrad: geometry not supported by the wgmma kernel");
  float* packed = nullptr;
  const size_t nb = conv_wgrad_packed_bytes(dW, co, ci, k);
  if (nb) {
    MYOLO_CHECK_CUDA(cudaMalloc(&packed, nb));
    MYOLO_CHECK_CUDA(cudaMemsetAsync(packed, 0, nb, s));
  }
  rc = launch_conv_wgrad_tc(xv, dv, k, stride, dil, dW, packed, co, ci, sms, s);
  cudaStreamSynchronize(s);
  if (packed) cudaFree(packed);
  return rc;
}

extern "C" int myolo_grads_check_finite(const float* grad, int64_t n, int32_t* found_inf, void* stream) {
  MYOLO_REQUIRE(grad && found_inf && n > 0, "grads_check_finite: bad arguments");
  int rc = check_device(nullptr);
  if (rc) return rc;
  return launch_grads_check_finite(grad, (long)n, found_inf, (cudaStream_t)stream);
}

extern "C" int myolo_sgd_step(float* param, float* grad, float* momentum_buf, const uint8_t* group, int64_t n, const float* lr,
                              const float* weight_decay, int n_groups, float momentum, int nesterov, const float* inv_scale,
                              const int32_t* found_inf, int zero_grad, void* stream) {
  NvtxRange nvtx_("myolo_sgd_step");
  int rc = check_device(nullptr);
  if (rc) return rc;
  return launch_sgd_step(param, grad, momentum_buf, group, (long)n, lr, weight_decay, n_groups, momentum, nesterov, inv_scale, found_inf,
                         zero_grad, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// gradient exchange: NCCL all-reduce of the flat gradient buffer, bound at run time from the libnccl already in the process
// ------------------------------------------------------------------------------------------------
#include <dlfcn.h>
typedef int (*PFN_ncclAllReduce)(const void*, void*, size_t, int /*ncclDataType_t*/, int /*ncclRedOp_t*/, void* /*ncclComm_t*/, cudaStream_t);
extern "C" int myolo_allreduce_grads(float* flat_grad, int64_t n, void* nccl_comm, void* stream) {
  NvtxRange nvtx_("myolo_allreduce_grads");
  MYOLO_REQUIRE(flat_grad && n > 0 && nccl_comm, "allreduce_grads: bad arguments");
  static PFN_ncclAllReduce fn = nullptr;
  if (!fn) {
    void* sym = dlsym(RTLD_DEFAULT, "ncclAllReduce");
    if (!sym) {
      void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
      if (h) sym = dlsym(h, "ncclAllReduce");
    }
    MYOLO_REQUIRE(sym, "allreduce_grads: no NCCL library is loaded in this process (torch.distributed with the nccl backend loads it)");
    fn = reinterpret_cast<PFN_ncclAllReduce>(sym);
  }
  const int rc = fn(flat_grad, flat_grad, (size_t)n, 7 /* ncclFloat32 */, 0 /* ncclSum */, nccl_comm, (cudaStream_t)stream);
  MYOLO_REQUIRE(rc == 0, "allreduce_grads: ncclAllReduce failed with ncclResult_t %d", rc);
  g_launch_count++;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// standalone fused conv (per-op parity tests, ncu captures)
// ------------------------------------------------------------------------------------------------
extern "C" int myolo_conv_bn_silu(const void* x, int B, int H, int W, int ci, const float* w, int co, int k, int stride, int dil,
                                  const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                                  const float* bias, int act, const void* residual, void* y, int path, void* stream) {
  MYOLO_REQUIRE(x && w && y && B > 0 && H > 0 && W > 0 && ci > 0 && co > 0, "conv_bn_silu: bad arguments");
  MYOLO_REQUIRE(ci % 16 == 0 && co % 8 == 0, "conv_bn_silu: standalone entry needs ci %% 16 == 0 and co %% 8 == 0");
  int sms = 0;
  int rc = check_device(&sms);
  if (rc) return rc;
  cudaStream_t s = (cudaStream_t)stream;
  const int co_pad = conv_n_pad(co), ci_pad = ci;
  __half* wp = nullptr;
  float* bp = nullptr;
  MYOLO_CHECK_CUDA(cudaMalloc(&wp, (size_t)co_pad * k * k * ci_pad * 2));
  MYOLO_CHECK_CUDA(cudaMalloc(&bp, (size_t)co_pad * 4));
  rc = pack_conv_weights(w, co, ci, k, gamma, beta, mean, var, eps, bias, wp, bp, co_pad, ci_pad, s);
  ConvOp c;
  const int pad = dil * (k / 2);
  const int ho = (H + 2 * pad - dil * (k - 1) - 1) / stride + 1, wo = (W + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  c.in = TensorView{const_cast<void*>(x), B, H, W, ci, ci, MYOLO_F16};
  c.out = TensorView{y, B, ho, wo, co, co, MYOLO_F16};
  c.has_res = residual != nullptr;
  if (c.has_res) c.res = TensorView{const_cast<void*>(residual), B, ho, wo, co, co, MYOLO_F16};
  c.k = k;
  c.stride = stride;
  c.dil = dil;
  c.act = act;
  c.w = wp;
  c.bias = bp;
  c.Ci_pad = ci_pad;
  c.Co_pad = co_pad;
  c.Co = co;
  if (!rc) {
    const bool elig = conv_tc_eligible(c);
    if ((path == 1 || path == 3) && !elig) {
      set_error("conv_bn_silu: shape not eligible for the tensor-core path");
      rc = MYOLO_E_INVALID;
    } else if (path == 2 || (path == 0 && !elig)) {
      rc = conv_simt_launch(c, s);
    } else {
      rc = conv_tc_prepare(c, sms);
      if (!rc) rc = conv_tc_launch(c, s);
    }
  }
  cudaError_t e = cudaStreamSynchronize(s);
  cudaFree(wp);
  cudaFree(bp);
  if (!rc && e != cudaSuccess) {
    set_error("conv_bn_silu: kernel failed: %s", cudaGetErrorString(e));
    rc = MYOLO_E_CUDA;
  }
  return rc;
}
