// C ABI + layer-plan executor: what Model.__init__/fuse() and Model.forward_once (reference models/yolo.py:293-316,339-347)
// become on the device.  The host-side planner (multiyolov5_b200/plan.py) lowers the module tree to a flat op list over
// liveness-packed NHWC buffers; this file resolves views, owns packed weights / tensor maps and replays the list on a stream.
#include <dlfcn.h>
#include <stdarg.h>

#include <algorithm>
#include <cmath>
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

int check_device(int* sms) {
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

// NCCL entry points, bound at run time from the libnccl already in the process (torch.distributed with the nccl backend loads it): the
// library does not link NCCL, so a process that never exchanges never needs it
static void* nccl_symbol(const char* name) {
  void* sym = dlsym(RTLD_DEFAULT, name);
  if (!sym) {
    void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD | RTLD_GLOBAL);
    if (h) sym = dlsym(h, name);
  }
  if (!sym) set_error("%s: no NCCL library is loaded in this process (torch.distributed with the nccl backend loads it)", name);
  return sym;
}
typedef int (*PFN_ncclAllReduce)(const void*, void*, size_t, int /*ncclDataType_t*/, int /*ncclRedOp_t*/, void* /*ncclComm_t*/, cudaStream_t);
typedef int (*PFN_ncclAllGather)(const void*, void*, size_t, int /*ncclDataType_t*/, void* /*ncclComm_t*/, cudaStream_t);
typedef int (*PFN_ncclCommQuery)(void* /*ncclComm_t*/, int*);
constexpr int kNcclFloat32 = 7, kNcclSum = 0;

static int nccl_allreduce_sum(float* buf, size_t n, void* comm, cudaStream_t s) {
  static PFN_ncclAllReduce fn = nullptr;
  if (!fn && !(fn = reinterpret_cast<PFN_ncclAllReduce>(nccl_symbol("ncclAllReduce")))) return MYOLO_E_INVALID;
  const int rc = fn(buf, buf, n, kNcclFloat32, kNcclSum, comm, s);
  MYOLO_REQUIRE(rc == 0, "ncclAllReduce failed with ncclResult_t %d", rc);
  g_launch_count++;
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
  bool owns_ws = true;            // false: ws / gws belong to the caller (myolo_plan_create_shared) and are never freed here
  std::vector<WeightSlot> slots;
  std::vector<ConvOp> convs;      // parallel to ops (valid for CONV ops)
  std::vector<int> conv_ready;    // tensor maps built
  int64_t last_launches = 0;
  bool force_simt = false;
  // CUDA-graph replay of the internal ops (everything that does not touch caller-owned tensors), captured in plan order as one chain.
  // lanes[0] is the capture origin, lanes[1] the backward's weight-gradient side lane; op_ev holds the backward's per-conv fork events and,
  // at n + 1, the join of the side lane.  Both are created by the first graph build.
  bool warmed = false, graph_dirty = true;
  std::vector<cudaStream_t> lanes;
  std::vector<cudaEvent_t> op_ev;
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
  // where the Detect decodes of the current call write z (myolo_plan_forward_pass): z_rows rows per image (0: the plan's own total), the
  // plan's rows from z_off on, box columns times z_inv, x mirrored at z_flip_w (0: none).  Read by the decodes only, which are never captured.
  int z_rows = 0, z_off = 0, z_flip_w = 0;
  float z_inv = 1.0f;
  // deferred running statistics (myolo_plan_set_defer_running / myolo_plan_apply_running)
  bool defer_running = false;
  RunningJob* d_run_jobs = nullptr;
  int n_run_jobs = 0;
  // synchronised BatchNorm (myolo_plan_set_bn_sync): an NCCL communicator, or one-GPU rank emulation over groups of images
  void* nccl_comm = nullptr;
  int sync_ranks = 0, sync_rank = 0;  // records per BN layer (world size / number of groups; 0: off) and this process's rank
  std::vector<int> sync_groups;       // rank emulation: images of each group, in rank order
  std::vector<float*> bn_sync;        // per BN op: [records (sync_ranks x (kBnRecHead + 2C)) | backward sums (sync_ranks x 2C) | 1 / N]
  unsigned long long seed = 0;       // dropout
  unsigned long long* d_step = nullptr;
  void* ce_scratch = nullptr;      // 16 bytes for the fused seg loss (valid-pixel count, loss sum)
  float* ce_gbuf = nullptr;        // per-pixel (softmax - onehot), NHWC fp32, of the fused seg loss
  size_t ce_gbuf_bytes = 0;
  void* ohem_ws = nullptr;         // the OHEM seg loss's selection state and per-pixel losses (ohem_scratch_bytes of B*H*W pixels)
  void* wf_ws = nullptr;           // the weighted / focal seg loss's sums and per-pixel factors (seg_wf_scratch_bytes of B*H*W pixels)
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

// shared_ws / shared_gws: caller-owned activation / gradient workspaces of shared_capacity bytes each (myolo_plan_create_shared), or
// null: the plan allocates (and frees) private ones
static int plan_create(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs, const int32_t* extra, int n_extra, int B,
                       int H, int W, int64_t workspace_bytes, int n_weight_slots, void* shared_ws, void* shared_gws,
                       int64_t shared_capacity, myolo_plan** out) {
  MYOLO_REQUIRE(ops && bufs && out && n_ops > 0 && n_bufs > 0 && B > 0 && H > 0 && W > 0, "plan_create: bad arguments");
  const bool shared = shared_ws != nullptr;
  if (shared) {
    MYOLO_REQUIRE(shared_gws && shared_capacity > 0, "plan_create_shared: null gradient workspace / capacity %lld",
                  (long long)shared_capacity);
    MYOLO_REQUIRE(reinterpret_cast<uintptr_t>(shared_ws) % 256 == 0 && reinterpret_cast<uintptr_t>(shared_gws) % 256 == 0,
                  "plan_create_shared: workspaces must be 256-byte aligned");
    MYOLO_REQUIRE(workspace_bytes > 0 && workspace_bytes <= shared_capacity,
                  "plan_create_shared: the plan needs %lld workspace bytes, the shared workspaces hold %lld", (long long)workspace_bytes,
                  (long long)shared_capacity);
  }
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
  cudaError_t e = cudaSuccess;
  if (shared) {              // the caller zeroes its workspaces (and re-zeroes them when another plan has written them)
    pl->ws = static_cast<unsigned char*>(shared_ws);
    pl->gws = static_cast<unsigned char*>(shared_gws);
    pl->owns_ws = false;
  } else {
    e = cudaMalloc(&pl->ws, workspace_bytes);
    if (e == cudaSuccess) e = cudaMemset(pl->ws, 0, workspace_bytes);
  }
  if (e == cudaSuccess && n_extra > 0) {
    e = cudaMalloc(&pl->d_extra, (size_t)n_extra * 4);
    if (e == cudaSuccess) e = cudaMemcpy(pl->d_extra, extra, (size_t)n_extra * 4, cudaMemcpyHostToDevice);
  }
  if (e != cudaSuccess) {
    set_error("plan_create: device allocation failed: %s", cudaGetErrorString(e));
    if (pl->ws && pl->owns_ws) cudaFree(pl->ws);
    if (pl->d_extra) cudaFree(pl->d_extra);
    delete pl;
    return MYOLO_E_CUDA;
  }
  pl->ws_bytes = workspace_bytes;
  *out = pl;
  return 0;
}

extern "C" int myolo_plan_create(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs, const int32_t* extra,
                                 int n_extra, int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, myolo_plan** out) {
  return plan_create(ops, n_ops, bufs, n_bufs, extra, n_extra, B, H, W, workspace_bytes, n_weight_slots, nullptr, nullptr, 0, out);
}

extern "C" int myolo_plan_create_shared(const myolo_op* ops, int n_ops, const myolo_buf_desc* bufs, int n_bufs, const int32_t* extra,
                                        int n_extra, int B, int H, int W, int64_t workspace_bytes, int n_weight_slots, void* ws, void* gws,
                                        int64_t capacity, myolo_plan** out) {
  MYOLO_REQUIRE(ws, "plan_create_shared: null activation workspace");
  return plan_create(ops, n_ops, bufs, n_bufs, extra, n_extra, B, H, W, workspace_bytes, n_weight_slots, ws, gws, capacity, out);
}

extern "C" void myolo_plan_destroy(myolo_plan* pl) {
  if (!pl) return;
  for (auto& s : pl->slots) {
    if (s.w) cudaFree(s.w);
    if (s.bias) cudaFree(s.bias);
  }
  if (pl->ws && pl->owns_ws) cudaFree(pl->ws);
  if (pl->d_extra) cudaFree(pl->d_extra);
  if (pl->decode_stream) cudaStreamDestroy(pl->decode_stream);
  if (pl->d_pack_jobs) cudaFree(pl->d_pack_jobs);
  if (pl->d_run_jobs) cudaFree(pl->d_run_jobs);
  if (pl->graph_exec) cudaGraphExecDestroy(pl->graph_exec);
  for (auto& e : pl->bwd_exec) if (e) cudaGraphExecDestroy(e);
  if (pl->graph) cudaGraphDestroy(pl->graph);
  for (auto e : pl->op_ev) cudaEventDestroy(e);
  for (auto& e : pl->ev_tail) if (e) cudaEventDestroy(e);
  for (auto st : pl->lanes) cudaStreamDestroy(st);
  for (auto& sl : pl->slots) {
    if (sl.w_dgrad) cudaFree(sl.w_dgrad);
    if (sl.zero_bias) cudaFree(sl.zero_bias);
  }
  for (auto p : pl->bn_stats) if (p) cudaFree(p);
  for (auto p : pl->bn_sync) if (p) cudaFree(p);
  if (pl->gws && pl->owns_ws) cudaFree(pl->gws);
  for (auto& sl : pl->slots) if (sl.dw_packed) cudaFree(sl.dw_packed);
  if (pl->tmp16) cudaFree(pl->tmp16);
  if (pl->ce_scratch) cudaFree(pl->ce_scratch);
  if (pl->d_step) cudaFree(pl->d_step);
  if (pl->ce_gbuf) cudaFree(pl->ce_gbuf);
  if (pl->ohem_ws) cudaFree(pl->ohem_ws);
  if (pl->wf_ws) cudaFree(pl->wf_ws);
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

// the extra table is read by the ops (and baked into captured graphs) at its device address: refreshed in place, in stream order
extern "C" int myolo_plan_set_extra(myolo_plan* pl, int offset, const void* src, int n, void* stream) {
  MYOLO_REQUIRE(pl && src && offset >= 0 && n > 0 && (size_t)offset + (size_t)n <= pl->extra.size(),
                "plan_set_extra: words [%d, %d) outside the extra table of %d words", offset, offset + n, pl ? (int)pl->extra.size() : 0);
  MYOLO_CHECK_CUDA(cudaMemcpyAsync(pl->d_extra + offset, src, (size_t)n * 4, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return 0;
}

// forward of one conv on resolved views (the plan's prepare_conv and myolo_conv_forward): the checks, the route (wgmma unless force_simt
// or conv_tc_eligible refuses) and, on the wgmma path, the tiling and tensor maps.  res: nullable.  An fp16 output view has the weights'
// co channels; an fp32 one at least co (the plan's fp32 head buffers carry co rounded up to 16), of which the conv writes the first co.
static int conv_forward_views(ConvOp& c, const TensorView& in, const TensorView& out, const TensorView* res, const WeightSlot& s, int k,
                              int stride, int dil, int act, bool force_simt, int num_sms) {
  c = ConvOp();
  c.in = in;
  c.out = out;
  c.has_res = res != nullptr;
  if (res) c.res = *res;
  c.k = k;
  c.stride = stride;
  c.dil = dil;
  c.act = act;
  c.w = s.w;
  c.bias = s.bias;
  c.Ci_pad = s.ci_pad;
  c.Co_pad = s.co_pad;
  c.Co = s.co;
  MYOLO_REQUIRE(s.k == k, "conv: kernel size %d != packed weights %d", k, s.k);
  MYOLO_REQUIRE(c.in.C == s.ci_pad, "conv: input view has %d channels, packed weights expect %d", c.in.C, s.ci_pad);
  MYOLO_REQUIRE(c.out.dtype == MYOLO_F32 ? c.out.C >= s.co : c.out.C == s.co, "conv: output view has %d channels, weights produce %d",
                c.out.C, s.co);
  MYOLO_REQUIRE(!res || (res->dtype == MYOLO_F16 && res->C >= s.co), "conv: the residual must be fp16 with %d channels", s.co);
  const int pad = dil * (k / 2);
  const int ho = (c.in.H + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  const int wo = (c.in.W + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  MYOLO_REQUIRE(ho == c.out.H && wo == c.out.W, "conv: output %dx%d does not match the view's %dx%d", ho, wo, c.out.H, c.out.W);
  c.use_tc = !force_simt && conv_tc_eligible(c);
  return c.use_tc ? conv_tc_prepare(c, num_sms) : 0;
}

static int prepare_conv(myolo_plan* pl, int i) {
  const myolo_op& op = pl->ops[i];
  MYOLO_REQUIRE(op.weight_slot >= 0 && op.weight_slot < (int)pl->slots.size(), "op %d: bad weight slot", i);
  const WeightSlot& s = pl->slots[op.weight_slot];
  if (!s.set) {
    set_error("op %d: weights of slot %d were never set (call myolo_plan_set_conv_weights first)", i, op.weight_slot);
    return MYOLO_E_STATE;
  }
  TensorView in, out, res;
  int rc;
  if ((rc = resolve_view(pl, op.in, &in))) return rc;
  if ((rc = resolve_view(pl, op.out, &out))) return rc;
  const bool has_res = op.in2.buf >= 0;
  if (has_res && (rc = resolve_view(pl, op.in2, &res))) return rc;
  if ((rc = conv_forward_views(pl->convs[i], in, out, has_res ? &res : nullptr, s, op.k, op.stride, op.dil, op.act, pl->force_simt,
                               pl->num_sms))) {
    const std::string msg = g_err;
    set_error("op %d: %s", i, msg.c_str());
    return rc;
  }
  pl->conv_ready[i] = 1;
  return 0;
}

// ---- synchronised BatchNorm: the exchanges of one BN op (myolo_plan_set_bn_sync) ----
static TensorView image_slice(TensorView v, int b0, int nb) {     // images [b0, b0 + nb) of a view
  v.base = static_cast<unsigned char*>(v.base) + (size_t)b0 * v.H * v.W * v.ctot * (v.dtype == MYOLO_F16 ? 2 : 4);
  v.B = nb;
  return v;
}
static size_t bn_rec_stride(int C) { return kBnRecHead + 2 * (size_t)C; }

// statistics of BN op i over all ranks: this rank's record (or each emulated group's), the all-gather, the combine into bn_stats[i]
static int bn_sync_forward(myolo_plan* pl, int i, const TensorView& in, const BnParams& bn, cudaStream_t s) {
  const int R = pl->sync_ranks, C = bn.C;
  const size_t stride = bn_rec_stride(C);
  if ((int)pl->bn_sync.size() <= i) pl->bn_sync.resize(pl->ops.size(), nullptr);
  if (!pl->bn_sync[i]) {
    const size_t n = (size_t)R * (stride + 2 * (size_t)C) + 4;
    MYOLO_CHECK_CUDA(cudaMalloc(&pl->bn_sync[i], n * sizeof(float)));
    MYOLO_CHECK_CUDA(cudaMemsetAsync(pl->bn_sync[i], 0, n * sizeof(float), s));
  }
  float* recs = pl->bn_sync[i];
  float* inv_n = recs + (size_t)R * (stride + 2 * (size_t)C);
  float* scratch = pl->bn_stats[i] + 2 * C;
  int rc;
  if (pl->nccl_comm) {
    static PFN_ncclAllGather gather = nullptr;
    if (!gather && !(gather = reinterpret_cast<PFN_ncclAllGather>(nccl_symbol("ncclAllGather")))) return MYOLO_E_INVALID;
    float* mine = recs + (size_t)pl->sync_rank * stride;
    if ((rc = launch_bn_stats_record(in, bn, mine, scratch, s))) return rc;
    // in place: NCCL's all-gather takes sendbuff == recvbuff + rank * count.  A byte copy: the int32 count travels exactly.
    const int nrc = gather(mine, recs, stride, kNcclFloat32, pl->nccl_comm, s);
    MYOLO_REQUIRE(nrc == 0, "bn sync: ncclAllGather failed with ncclResult_t %d", nrc);
    g_launch_count++;
  } else {
    for (int g = 0, b0 = 0; g < R; b0 += pl->sync_groups[g++])
      if ((rc = launch_bn_stats_record(image_slice(in, b0, pl->sync_groups[g]), bn, recs + g * stride, scratch, s))) return rc;
  }
  return launch_bn_sync_combine(recs, R, bn, pl->bn_stats[i], inv_n, s);
}

// backward of BN op i over all ranks: local {sum dz, sum dz*xhat} (this rank's, or each group's), their sum over ranks, then dx with the
// global sums and 1 / N.  d_gamma / d_beta take the LOCAL sums: the flat-gradient all-reduce averages them, as DDP does.
static int bn_sync_backward(myolo_plan* pl, int i, const TensorView& u, const TensorView& dy, const TensorView& du, const TensorView* d_res,
                            const BnParams& bn, int act, cudaStream_t s) {
  MYOLO_REQUIRE(i < (int)pl->bn_sync.size() && pl->bn_sync[i], "backward: BN op %d has no synchronised forward", i);
  const int R = pl->sync_ranks, C = bn.C;
  float* sums = pl->bn_sync[i] + (size_t)R * bn_rec_stride(C);
  const float* inv_n = sums + (size_t)R * 2 * C;
  float* scratch = pl->bn_stats[i] + 2 * C;
  int rc;
  if (pl->nccl_comm) {
    if ((rc = launch_bn_bwd_sums(u, dy, bn, pl->bn_stats[i], act, scratch, sums, s))) return rc;
    if ((rc = nccl_allreduce_sum(sums, 2 * (size_t)C, pl->nccl_comm, s))) return rc;
  } else {
    for (int g = 0, b0 = 0; g < R; b0 += pl->sync_groups[g++])
      if ((rc = launch_bn_bwd_sums(image_slice(u, b0, pl->sync_groups[g]), image_slice(dy, b0, pl->sync_groups[g]), bn, pl->bn_stats[i], act,
                                   scratch, sums + (size_t)g * 2 * C, s)))
        return rc;
    if ((rc = launch_bn_sync_sum(sums, R, 2 * C, s))) return rc;
  }
  return launch_bn_act_bwd(u, dy, du, d_res, bn, pl->bn_stats[i], act, scratch, s, sums, inv_n);
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
      if (pl->sync_ranks) rc = bn_sync_forward(pl, i, in, bn, s);
      else rc = launch_bn_stats(in, bn, pl->bn_stats[i], pl->bn_stats[i] + 2 * bn.C, s, pl->defer_running);
      if (rc) return rc;
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
                                  raw ? raw[level] : nullptr, z, pl->z_off + op.aux[3], pl->z_rows > 0 ? pl->z_rows : op.aux[4], s, pl->z_inv,
                                  pl->z_flip_w);
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
// graph capture of the internal ops
// ------------------------------------------------------------------------------------------------
static bool is_external_op(int kind) {
  return kind == MYOLO_OP_INPUT_FOCUS || kind == MYOLO_OP_DETECT_DECODE || kind == MYOLO_OP_SEG_UPSAMPLE;
}

// The forward graph is ONE chain of the internal ops in plan order.  Every conv launch fills the machine, so branch concurrency buys
// little, while a capture over several streams makes the graph runtime spread the nodes over many internal streams: every edge becomes a
// cross-stream dependency and the programmatic-dependent-launch edges between consecutive convs are lost.
static int build_graph(myolo_plan* pl) {
  const int n = (int)pl->ops.size();
  if (pl->lanes.empty()) {
    pl->lanes.resize(2);
    for (auto& st : pl->lanes) MYOLO_CHECK_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    pl->op_ev.resize(n + 2);
    for (auto& e : pl->op_ev) MYOLO_CHECK_CUDA(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  }
  if (pl->graph_exec) { cudaGraphExecDestroy(pl->graph_exec); pl->graph_exec = nullptr; }
  if (pl->graph) { cudaGraphDestroy(pl->graph); pl->graph = nullptr; }
  cudaStream_t origin = pl->lanes[0];
  MYOLO_CHECK_CUDA(cudaStreamBeginCapture(origin, cudaStreamCaptureModeThreadLocal));
  int rc = 0, count = 0;
  for (int i = 0; i < n; ++i) {
    if (is_external_op(pl->ops[i].kind)) continue;
    if ((rc = run_op(pl, i, nullptr, 0, nullptr, nullptr, nullptr, 0, nullptr, origin))) break;
    ++count;
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
  if (!pl->warmed || pl->sync_ranks) {
    // first call (lazy tensor-map / attribute setup happens here): plain in-order replay.  A plan with synchronised BatchNorm always runs
    // so: its NCCL exchanges are never captured into a graph (torch's communicator is used eagerly for the flat gradients as well)
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
    if (pl->ops[i].kind == MYOLO_OP_INPUT_FOCUS) {
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

extern "C" int myolo_plan_forward_pass(myolo_plan* pl, const void* x, int x_dtype, float* z, int z_rows_total, int z_row_offset,
                                       float z_inv_scale, int z_flip_w, void* seg, int seg_dtype, int64_t* seg_argmax, void* stream) {
  MYOLO_REQUIRE(pl && x && z, "plan_forward_pass: null plan / input / z");
  int plan_rows = 0;
  for (const auto& op : pl->ops)
    if (op.kind == MYOLO_OP_DETECT_DECODE) plan_rows = op.aux[4];
  MYOLO_REQUIRE(plan_rows > 0, "plan_forward_pass: the plan has no Detect decode");
  MYOLO_REQUIRE(z_row_offset >= 0 && z_rows_total >= plan_rows && z_row_offset <= z_rows_total - plan_rows,
                "plan_forward_pass: rows [%d, %d) of the plan's outputs do not fit in %d rows", z_row_offset, z_row_offset + plan_rows,
                z_rows_total);
  MYOLO_REQUIRE(z_inv_scale > 0.f && std::isfinite(z_inv_scale), "plan_forward_pass: inv_scale %g", z_inv_scale);
  MYOLO_REQUIRE(z_flip_w >= 0, "plan_forward_pass: flip width %d", z_flip_w);
  pl->z_rows = z_rows_total;
  pl->z_off = z_row_offset;
  pl->z_inv = z_inv_scale;
  pl->z_flip_w = z_flip_w;
  const int rc = myolo_plan_forward(pl, x, x_dtype, z, nullptr, seg, seg_dtype, seg_argmax, stream);
  pl->z_rows = pl->z_off = pl->z_flip_w = 0;
  pl->z_inv = 1.0f;
  return rc;
}

// The low-res logits stay valid after a forward: the planner keeps whatever the external ops read live to the end of the plan, and an
// inference plan owns its workspace, so another member's launches never write there.
extern "C" int myolo_seg_ensemble(myolo_plan* const* plans, int K, void* seg, int seg_dtype, int64_t* seg_argmax, void* stream) {
  NvtxRange nvtx_("myolo_seg_ensemble");
  MYOLO_REQUIRE(plans && K >= 1 && K <= MYOLO_ENSEMBLE_MAX, "seg_ensemble: %d members (1..%d)", K, MYOLO_ENSEMBLE_MAX);
  MYOLO_REQUIRE(seg || seg_argmax, "seg_ensemble: no output");
  MYOLO_REQUIRE(!seg || seg_dtype == MYOLO_F16 || seg_dtype == MYOLO_F32, "seg_ensemble: seg dtype %d", seg_dtype);
  int rc = check_device(nullptr);
  if (rc) return rc;
  TensorView ins[MYOLO_ENSEMBLE_MAX];
  int n_cls = 0;
  for (int k = 0; k < K; ++k) {
    const myolo_plan* pl = plans[k];
    MYOLO_REQUIRE(pl, "seg_ensemble: member %d has no plan", k);
    const myolo_op* up = nullptr;
    for (const auto& op : pl->ops)
      if (op.kind == MYOLO_OP_SEG_UPSAMPLE && op.aux[1] == 0) up = &op;
    MYOLO_REQUIRE(up, "seg_ensemble: member %d's plan has no seg output", k);
    MYOLO_REQUIRE(pl->B == plans[0]->B && pl->H == plans[0]->H && pl->W == plans[0]->W,
                  "seg_ensemble: member %d's plan is %dx%dx%d, member 0's %dx%dx%d", k, pl->B, pl->H, pl->W, plans[0]->B, plans[0]->H,
                  plans[0]->W);
    MYOLO_REQUIRE(k == 0 || up->aux[0] == n_cls, "seg_ensemble: member %d has %d seg classes, member 0 %d", k, up->aux[0], n_cls);
    n_cls = up->aux[0];
    if ((rc = resolve_view(pl, up->in, &ins[k]))) return rc;
  }
  return launch_seg_ensemble(ins, K, n_cls, plans[0]->H, plans[0]->W, seg, seg_dtype, seg_argmax, (cudaStream_t)stream);
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

static void conv_info_slots(const ConvOp& c, int32_t* info) {
  for (int i = 0; i < 12; ++i) info[i] = 0;
  info[0] = c.use_tc ? 1 : 0;
  if (c.use_tc) {
    info[1] = c.grid; info[2] = c.smem; info[3] = c.p.BN; info[4] = c.p.num_stages; info[5] = c.p.strip;
    info[6] = c.p.resident; info[7] = 1; info[8] = c.p.total_tiles; info[9] = c.p.n_tiles_n; info[10] = c.p.kc;
    info[11] = c.ctas_per_sm;
  }
}

// which kernel a conv op of the plan takes and how it is tiled (valid after the first forward): info[0..11] =
// {1 wgmma / 0 CUDA-core, grid, dynamic smem bytes, BN, pipeline stages, mode (0: one TMA box per tap, 1: one strip per filter row),
//  weights-stationary (1: the CTA keeps its weight slice in shared memory),
//  tiles per accumulator round (always 1), total tiles, n tiles in N, kc, CTAs per SM (1 or 2)}
extern "C" int myolo_plan_conv_info(myolo_plan* pl, int op_index, int32_t* info) {
  MYOLO_REQUIRE(pl && info && op_index >= 0 && op_index < (int)pl->ops.size(), "conv_info: bad arguments");
  MYOLO_REQUIRE(pl->ops[op_index].kind == MYOLO_OP_CONV, "conv_info: op %d is not a conv", op_index);
  int rc;
  if (!pl->conv_ready[op_index] && (rc = prepare_conv(pl, op_index))) return rc;
  conv_info_slots(pl->convs[op_index], info);
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
  MYOLO_REQUIRE(!defer || !pl->sync_ranks, "set_defer_running: the plan synchronises its BatchNorm statistics across ranks");
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

extern "C" int myolo_plan_set_bn_sync(myolo_plan* pl, void* nccl_comm, const int32_t* rank_images, int n_groups) {
  MYOLO_REQUIRE(pl, "set_bn_sync: null plan");
  MYOLO_REQUIRE(!(nccl_comm && rank_images), "set_bn_sync: an NCCL communicator or rank emulation, not both");
  int ranks = 0, rank = 0;
  std::vector<int> groups;
  if (nccl_comm) {
    auto count = reinterpret_cast<PFN_ncclCommQuery>(nccl_symbol("ncclCommCount"));
    auto user_rank = reinterpret_cast<PFN_ncclCommQuery>(nccl_symbol("ncclCommUserRank"));
    if (!count || !user_rank) return MYOLO_E_INVALID;
    MYOLO_REQUIRE(count(nccl_comm, &ranks) == 0 && user_rank(nccl_comm, &rank) == 0 && ranks >= 1 && rank >= 0 && rank < ranks,
                  "set_bn_sync: cannot query the NCCL communicator");
  } else if (rank_images) {
    MYOLO_REQUIRE(n_groups >= 1, "set_bn_sync: %d image groups", n_groups);
    int total = 0;
    for (int g = 0; g < n_groups; ++g) {
      MYOLO_REQUIRE(rank_images[g] >= 1, "set_bn_sync: group %d has %d images", g, rank_images[g]);
      total += rank_images[g];
      groups.push_back(rank_images[g]);
    }
    MYOLO_REQUIRE(total == pl->B, "set_bn_sync: the groups hold %d images, the plan's batch is %d", total, pl->B);
    ranks = n_groups;
  }
  MYOLO_REQUIRE(!ranks || !pl->defer_running, "set_bn_sync: the plan defers its running statistics (myolo_plan_set_defer_running)");
  if (ranks != pl->sync_ranks) {        // the buffers hold one record per rank
    for (auto& p : pl->bn_sync) if (p) { cudaFree(p); p = nullptr; }
  }
  pl->nccl_comm = nccl_comm;
  pl->sync_ranks = ranks;
  pl->sync_rank = rank;
  pl->sync_groups = groups;
  pl->graph_dirty = true;               // the BN launches of captured graphs are the unsynchronised ones
  pl->bwd_dirty = true;
  return 0;
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

extern "C" int myolo_plan_train_forward_multi(myolo_plan* pl, const void* x, int x_dtype, float* const* raw, float* const* seg, void* stream) {
  NvtxRange nvtx_("myolo_plan_train_forward_multi");
  MYOLO_REQUIRE(pl && x, "train_forward: null plan / input");
  pl->seg_outs[1] = seg ? seg[1] : nullptr;
  pl->seg_outs[2] = seg ? seg[2] : nullptr;
  if (!pl->d_step) {
    MYOLO_CHECK_CUDA(cudaMalloc(&pl->d_step, sizeof(unsigned long long)));
    MYOLO_CHECK_CUDA(cudaMemset(pl->d_step, 0, sizeof(unsigned long long)));
  }
  {   // a new dropout mask per forward; the counter lives on the device so that captured graphs see the new value
    int brc = launch_bump_step(pl->d_step, (cudaStream_t)stream);
    if (brc) return brc;
  }
  // same executor as inference: first call in order (lazy allocations / tensor maps), then CUDA-graph replay of the internal
  // ops with the input conversion before and the caller-owned outputs (raw x_i, seg logits) after the graph
  int rc = myolo_plan_forward(pl, x, x_dtype, nullptr, raw, seg ? seg[0] : nullptr, MYOLO_F32, nullptr, stream);
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

// which kernels the backward of one conv takes (myolo_conv_backward's info slots 0-2)
enum { kDgradNone = 0, kDgradSmall = 1, kDgradWgmma = 2, kDgradSimt = 3 };
enum { kWgradSmall = 1, kWgradMma = 2, kWgradWgmmaDirect = 3, kWgradWgmmaPacked = 4 };

// tiny maps / fp32 inputs: generic kernels on the fp32 master weights
static bool conv_bwd_small(const TensorView& xin, const TensorView& gout) {
  return xin.dtype == MYOLO_F32 || (long)gout.B * gout.H * gout.W <= 1024 || gout.H * gout.W < 128;
}

// fp16 scratch of the backward of one conv: dY cast from fp32 (head gradients) at 0, the zero-stuffed stride-2 dY at *stuffed_off
static size_t conv_bwd_tmp16_bytes(const TensorView& xin, const TensorView& gout, int co, int stride, size_t* stuffed_off) {
  if (conv_bwd_small(xin, gout)) return 0;
  const int cpad = (int)align_up(co, 16);
  size_t need = 0;
  if (gout.dtype == MYOLO_F32) need = (size_t)gout.B * gout.H * gout.W * cpad * 2;
  if (stuffed_off) *stuffed_off = align_up((int64_t)need, 256);
  if (stride == 2) need = align_up((int64_t)need, 256) + (size_t)gout.B * (2 * gout.H) * (2 * gout.W) * cpad * 2;
  return need;
}

// the scratch the backward of one conv works in: the fp16 dY scratch (at least conv_bwd_tmp16_bytes) and the data-gradient conv, whose
// tensor maps (built once, *dconv_ready) point into tmp16 and grad(in)
struct ConvBwdScratch {
  __half* tmp16;
  ConvOp* dconv;
  int* dconv_ready;
};

// backward of one conv on resolved views: dY = gout; grad(in) += conv^T(dY, W) when gin is given; dW += ...; dbias += ...
// `ws`: stream of the weight / bias gradient kernels, forked from s at `fork` (null: they stay on s).  Nothing downstream in the backward
// pass reads them, so the plan's walk forks them onto a side lane where they overlap the latency-bound chain of data-gradient / BN kernels;
// the caller joins the lane at the end.  info (nullable, 16 slots): see myolo_conv_backward in include/myolo.h.
static int conv_backward_views(const TensorView& xin, const TensorView& gout, const TensorView* gin, WeightSlot& sl, int k, int stride,
                               int dil, const ConvBwdScratch& scr, int num_sms, bool force_simt, bool no_wgrad_tc, cudaStream_t s,
                               cudaStream_t ws, cudaEvent_t fork, bool* used_side, int32_t* info) {
  int rc;
  if (info)
    for (int j = 0; j < 16; ++j) info[j] = 0;
  if (conv_bwd_small(xin, gout)) {
    TensorView gy = gout;
    gy.C = sl.co;
    if (info) {
      info[0] = gin ? kDgradSmall : kDgradNone;
      info[1] = kWgradSmall;
      info[2] = sl.d_bias ? (gout.dtype == MYOLO_F32 ? 1 : 2) : 0;
    }
    return launch_conv_small_bwd(xin, gy, gin, sl.w_master, sl.d_w, sl.d_bias, sl.co, sl.ci, k, stride, dil, s);
  }
  // dY in fp16 (cast fp32 head gradients; zero-stuff for stride 2)
  const int cpad = (int)align_up(sl.co, 16);
  TensorView dy16 = gout;
  size_t stuffed_off = 0;
  conv_bwd_tmp16_bytes(xin, gout, sl.co, stride, &stuffed_off);
  const bool s2 = stride == 2;
  if (gout.dtype == MYOLO_F32) {
    dy16 = TensorView{scr.tmp16, gout.B, gout.H, gout.W, cpad, cpad, MYOLO_F16};
    if ((rc = launch_cast_f32_to_f16(gout, dy16, s))) return rc;
  } else {
    MYOLO_REQUIRE(gout.C == sl.co && sl.co % 16 == 0, "conv backward: fp16 conv gradient needs Co %% 16 == 0 (Co=%d)", sl.co);
  }
  // weight / bias gradients
  // dY in the shared fp16 scratch (fp32 head gradients) is overwritten by the next conv: those few layers stay on the main stream
  cudaStream_t wst = (fork && ws != s && gout.dtype != MYOLO_F32) ? ws : s;
  if (wst != s) {
    MYOLO_CHECK_CUDA(cudaEventRecord(fork, s));          // dY (and everything before it on the main chain) is final here
    MYOLO_CHECK_CUDA(cudaStreamWaitEvent(wst, fork, 0));
    *used_side = true;
  }
  if (!no_wgrad_tc && conv_wgrad_tc_eligible(xin, dy16, k, stride, dil, sl.co, sl.ci)) {
    const size_t nb = conv_wgrad_packed_bytes(sl.d_w, sl.co, sl.ci, k);
    if (!sl.dw_packed && nb) {
      MYOLO_CHECK_CUDA(cudaMalloc(&sl.dw_packed, nb));
      MYOLO_CHECK_CUDA(cudaMemset(sl.dw_packed, 0, nb));
    }
    if (info) info[1] = nb ? kWgradWgmmaPacked : kWgradWgmmaDirect;
    if ((rc = launch_conv_wgrad_tc(xin, dy16, k, stride, dil, sl.d_w, sl.dw_packed, sl.co, sl.ci, num_sms, wst, info ? info + 8 : nullptr)))
      return rc;
  } else {
    if (info) info[1] = kWgradMma;
    if ((rc = launch_conv_wgrad(xin, dy16, k, stride, dil, sl.d_w, sl.co, sl.ci, nullptr, wst))) return rc;
  }
  if (sl.d_bias) {   // the bias gradient of an fp32 head gradient is summed from the fp32 values, not from their fp16 cast
    TensorView gy = gout.dtype == MYOLO_F32 ? gout : dy16;
    gy.C = sl.co;
    if (info) info[2] = gy.dtype == MYOLO_F32 ? 1 : 2;
    if ((rc = launch_bias_grad(gy, sl.d_bias, sl.co, wst))) return rc;
  }
  if (!gin) return 0;
  // data gradient = stride-1 conv of (zero-stuffed) dY with flipped / transposed weights, accumulated into grad(in).  Its N tile (sl.ci
  // rounded up to 16 channels, or a multiple of 16 dividing that: conv_tc_prepare) never reaches past the padded pack.
  const int n_pad = (int)align_up(sl.ci, 16);
  if (!sl.w_dgrad) {
    MYOLO_CHECK_CUDA(cudaMalloc(&sl.w_dgrad, (size_t)n_pad * k * k * cpad * 2));
    MYOLO_CHECK_CUDA(cudaMalloc(&sl.zero_bias, (size_t)n_pad * 4));
  }
  if (!sl.dgrad_valid) {   // (first use; later refreshes happen in refresh_dgrad_packs, outside any captured graph)
    if ((rc = pack_dgrad_weights(sl.w_master, sl.co, sl.ci, k, sl.w_dgrad, sl.zero_bias, n_pad, cpad, s))) return rc;
    sl.dgrad_valid = true;
    sl.dgrad_n_pad = n_pad;
    sl.dgrad_cpad = cpad;
  }
  TensorView din = dy16;
  if (s2) {
    din = TensorView{reinterpret_cast<unsigned char*>(scr.tmp16) + stuffed_off, gout.B, 2 * gout.H, 2 * gout.W, cpad, cpad, MYOLO_F16};
    TensorView src = dy16;
    src.C = cpad;
    if (gout.dtype != MYOLO_F32) { src = gout; }
    MYOLO_REQUIRE(src.C == cpad, "conv backward: stride-2 gradient channel padding mismatch");
    if ((rc = launch_zero_stuff2(src, din, s))) return rc;
  }
  ConvOp& c = *scr.dconv;
  if (!*scr.dconv_ready) {
    c = ConvOp();
    c.in = din;
    c.in.C = cpad;
    c.out = *gin;
    c.out.C = sl.ci;
    c.has_res = true;
    c.res = c.out;
    c.k = k;
    c.stride = 1;
    c.dil = dil;
    c.act = MYOLO_ACT_NONE;
    c.w = sl.w_dgrad;
    c.bias = sl.zero_bias;
    c.Ci_pad = cpad;
    c.Co_pad = n_pad;
    c.Co = sl.ci;
    MYOLO_REQUIRE(din.H == gin->H && din.W == gin->W, "conv backward: data-gradient geometry %dx%d vs %dx%d", din.H, din.W, gin->H, gin->W);
    c.use_tc = !force_simt && conv_tc_eligible(c);
    if (c.use_tc && (rc = conv_tc_prepare(c, num_sms))) return rc;
    *scr.dconv_ready = 1;
  }
  if (info) {
    info[0] = c.use_tc ? kDgradWgmma : kDgradSimt;
    if (c.use_tc) {
      info[3] = c.p.kc; info[4] = c.p.BN; info[5] = c.ctas_per_sm; info[6] = c.p.resident; info[7] = c.p.strip;
      info[13] = c.p.n_tiles_n; info[14] = c.Co_pad;
    }
  }
  return c.use_tc ? conv_tc_launch(c, s) : conv_simt_launch(c, s);
}

// backward of one conv op of the plan on its views in the activation / gradient workspaces
static int conv_backward(myolo_plan* pl, int i, bool need_dgrad, cudaStream_t s, cudaStream_t ws, bool* used_side) {
  const myolo_op& op = pl->ops[i];
  WeightSlot& sl = pl->slots[op.weight_slot];
  MYOLO_REQUIRE(sl.set && sl.w_master && sl.d_w, "op %d: conv slot %d has no master weights / gradient pointer", i, op.weight_slot);
  TensorView xin, gout, gin;
  int rc;
  if ((rc = resolve_view(pl, op.in, &xin)) || (rc = grad_view(pl, op.out, &gout)) || (rc = grad_view(pl, op.in, &gin))) return rc;
  const size_t need = conv_bwd_tmp16_bytes(xin, gout, sl.co, op.stride, nullptr);
  if (need && (rc = ensure_tmp16(pl, need))) return rc;
  if (pl->dconvs.size() != pl->ops.size()) { pl->dconvs.resize(pl->ops.size()); pl->dconv_ready.assign(pl->ops.size(), 0); }
  const bool had_pack = sl.w_dgrad != nullptr;
  const ConvBwdScratch scr{pl->tmp16, &pl->dconvs[i], &pl->dconv_ready[i]};
  cudaEvent_t fork = (ws != s && (int)pl->op_ev.size() > i) ? pl->op_ev[i] : nullptr;
  rc = conv_backward_views(xin, gout, need_dgrad ? &gin : nullptr, sl, op.k, op.stride, op.dil, scr, pl->num_sms, pl->force_simt, false, s,
                           ws, fork, used_side, nullptr);
  if (!had_pack && sl.w_dgrad) pl->pack_table_dirty = true;   // the grouped repack refreshes the new data-gradient pack from now on
  return rc;
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
  if (!pl->bwd_warm[mask] || pl->sync_ranks) {
    // first backward with this seed set: in order on the caller's stream (allocations, tensor maps, weight packs happen here); always
    // with synchronised BatchNorm, whose exchanges are not captured (myolo_plan_forward)
    rc = backward_walk(pl, live, s, &n_ops);
    if (!rc && !pl->bwd_dirty) pl->bwd_warm[mask] = true;
    return rc;
  }
  if (!pl->bwd_exec[mask]) {
    if (pl->lanes.empty()) { set_error("backward: forward graph state missing"); return MYOLO_E_INVALID; }
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

static int plan_backward(myolo_plan* pl, const float* const* grad_raw, const float* grad_seg, void* stream) {
  MYOLO_REQUIRE(pl->train_fwd_done, "backward: call myolo_plan_train_forward_multi first");
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

extern "C" int myolo_plan_backward_multi(myolo_plan* pl, const float* const* grad_raw, const float* const* grad_seg, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward_multi");
  MYOLO_REQUIRE(pl, "backward: null plan");
  pl->grad_segs[1] = grad_seg ? grad_seg[1] : nullptr;
  pl->grad_segs[2] = grad_seg ? grad_seg[2] : nullptr;
  int rc = plan_backward(pl, grad_raw, grad_seg ? grad_seg[0] : nullptr, stream);
  pl->grad_segs[1] = pl->grad_segs[2] = nullptr;
  return rc;
}

// fused seg loss (SURVEY.md section 8f rank 3): CE(ignore_index) of the x8-upsampled logits of the last train forward is evaluated and
// differentiated straight from the low-resolution logits; the backward then runs as the seg pass (seed mask 8)
// ohem: OhemCELoss(thresh) with thresh_t = -log(thresh) instead of the mean CE; wf: the class-weighted CE / focal loss (weights, gamma)
static int backward_seg_fused(myolo_plan* pl, const int64_t* labels, int ignore_index, float factor, const float* scale_dev, float* loss_out,
                              cudaStream_t s, bool ohem, float thresh_t, bool wf = false, const float* weights = nullptr, float gamma = 0.f) {
  MYOLO_REQUIRE(pl && pl->train_fwd_done && labels, "backward_seg_ce: call myolo_plan_train_forward_multi first / null labels");
  if (!pl->gws) MYOLO_CHECK_CUDA(cudaMalloc(&pl->gws, pl->ws_bytes));
  MYOLO_CHECK_CUDA(cudaMemsetAsync(pl->gws, 0, pl->ws_bytes, s));
  if (!pl->ce_scratch) MYOLO_CHECK_CUDA(cudaMalloc(&pl->ce_scratch, 16));
  if (ohem && !pl->ohem_ws) MYOLO_CHECK_CUDA(cudaMalloc(&pl->ohem_ws, ohem_scratch_bytes((long)pl->B * pl->H * pl->W)));   // the plan's shape is fixed
  if (wf && !pl->wf_ws) MYOLO_CHECK_CUDA(cudaMalloc(&pl->wf_ws, seg_wf_scratch_bytes((long)pl->B * pl->H * pl->W)));
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
      if (wf)
        rc = launch_seg_wf_fused(lo, op.aux[0], reinterpret_cast<const long long*>(labels), pl->H, pl->W, ignore_index, dlo, factor,
                                 scale_dev, pl->ce_gbuf, pl->wf_ws, weights, gamma, loss_out, s);
      else
        rc = launch_seg_ce_fused(lo, op.aux[0], reinterpret_cast<const long long*>(labels), pl->H, pl->W, ignore_index, dlo, factor,
                                 scale_dev, pl->ce_scratch, pl->ce_gbuf, loss_out, s, ohem ? pl->ohem_ws : nullptr, thresh_t);
      break;
    }
  if (rc) { if (rc == MYOLO_E_INVALID) set_error("backward_seg_ce: the plan has no segmentation output"); return rc; }
  return backward_run(pl, 8, live, s);
}

extern "C" int myolo_plan_backward_seg_ce(myolo_plan* pl, const int64_t* labels, int ignore_index, float factor, const float* scale_dev,
                                          float* loss_out, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward_seg_ce");
  return backward_seg_fused(pl, labels, ignore_index, factor, scale_dev, loss_out, (cudaStream_t)stream, false, 0.f);
}

extern "C" int myolo_plan_backward_seg_ohem(myolo_plan* pl, const int64_t* labels, int ignore_index, float thresh_t, float factor,
                                            const float* scale_dev, float* loss_out, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward_seg_ohem");
  return backward_seg_fused(pl, labels, ignore_index, factor, scale_dev, loss_out, (cudaStream_t)stream, true, thresh_t);
}

extern "C" int myolo_plan_backward_seg_loss(myolo_plan* pl, const int64_t* labels, int ignore_index, const float* class_weights, float gamma,
                                            float factor, const float* scale_dev, float* loss_out, void* stream) {
  NvtxRange nvtx_("myolo_plan_backward_seg_loss");
  return backward_seg_fused(pl, labels, ignore_index, factor, scale_dev, loss_out, (cudaStream_t)stream, false, 0.f, true, class_weights,
                            gamma);
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
  // weight-gradient lane (exists once the forward graph has created the plan's streams / events)
  cudaStream_t side = (pl->lanes.size() >= 2 && pl->lanes[1] != s && (int)pl->op_ev.size() >= n + 2) ? pl->lanes[1] : s;
  bool used_side = false;
  for (int i = n - 1; i >= 0 && !rc; --i) {
    const myolo_op& op = pl->ops[i];
    TensorView a, b, c, d;
    if (op.kind == MYOLO_OP_SEG_UPSAMPLE || op.kind == MYOLO_OP_DETECT_DECODE || op.kind == MYOLO_OP_INPUT_FOCUS) continue;
    if (!is_live(op.out)) continue;
    mark(op.in);
    mark(op.in2);
    ++*n_ops;
    switch (op.kind) {
      case MYOLO_OP_CONV:
        rc = conv_backward(pl, i, !is_input_buf[op.in.buf], s, side, &used_side);
        break;
      case MYOLO_OP_BN_ACT: {
        const bool has_res = op.in2.buf >= 0;
        if ((rc = resolve_view(pl, op.in, &a)) || (rc = grad_view(pl, op.out, &b)) || (rc = grad_view(pl, op.in, &c))) break;
        if (has_res && (rc = grad_view(pl, op.in2, &d))) break;
        const BnParams& bn = pl->bns[op.aux[0]];
        // synchronised BN: one all-reduce per live BN op.  NCCL needs the same sequence of collectives on every rank; every rank runs
        // the same op list (built from the same model), and which ops are live depends only on the seed mask, not on the data
        if (pl->sync_ranks) rc = bn_sync_backward(pl, i, a, b, c, has_res ? &d : nullptr, bn, op.act, s);
        else rc = launch_bn_act_bwd(a, b, c, has_res ? &d : nullptr, bn, pl->bn_stats[i], op.act, pl->bn_stats[i] + 2 * bn.C, s);
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
  }
  if (used_side) {   // join the weight-gradient lane (required to close a capture; in eager mode it orders the optimiser after it)
    if (cudaEventRecord(pl->op_ev[n + 1], side) != cudaSuccess || cudaStreamWaitEvent(s, pl->op_ev[n + 1], 0) != cudaSuccess) {
      if (!rc) { set_error("backward: joining the weight-gradient lane failed"); rc = MYOLO_E_CUDA; }
    }
  }
  return rc;
}

extern "C" int myolo_conv_backward(const void* x, int x_dtype, int B, int H, int W, int x_ctot, int x_coff, const void* dy, int dy_dtype,
                                   int dy_ctot, int dy_coff, void* gin, int gin_ctot, int gin_coff, const float* w, int co, int ci, int k,
                                   int stride, int dil, float* dW, float* dbias, int route, int32_t* info, void* stream) {
  NvtxRange nvtx_("myolo_conv_backward");
  MYOLO_REQUIRE(x && dy && w && dW && B > 0 && H > 0 && W > 0 && co > 0 && ci > 0 && k >= 1 && k % 2 == 1 && (stride == 1 || stride == 2) &&
                dil >= 1 && (route & ~(MYOLO_CONV_BWD_SIMT | MYOLO_CONV_BWD_NO_WGRAD_TC)) == 0, "conv_backward: bad arguments");
  MYOLO_REQUIRE((x_dtype == MYOLO_F16 || x_dtype == MYOLO_F32) && (dy_dtype == MYOLO_F16 || dy_dtype == MYOLO_F32),
                "conv_backward: x and dy must be MYOLO_F16 or MYOLO_F32");
  // the plan's views: x and grad(in) carry ci rounded up to 16 channels; an fp32 head gradient carries co rounded up to 16 (zero padding)
  const int xc = (int)align_up(ci, 16), dyc = dy_dtype == MYOLO_F32 ? (int)align_up(co, 16) : co;
  MYOLO_REQUIRE(x_coff >= 0 && x_coff + xc <= x_ctot && dy_coff >= 0 && dy_coff + dyc <= dy_ctot &&
                (!gin || (gin_coff >= 0 && gin_coff + xc <= gin_ctot)), "conv_backward: channel slice outside its buffer");
  int sms = 0;
  int rc = check_device(&sms);
  if (rc) return rc;
  const int pad = dil * (k / 2);
  const int Ho = (H + 2 * pad - dil * (k - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  MYOLO_REQUIRE(Ho > 0 && Wo > 0, "conv_backward: empty output map");
  const size_t xes = x_dtype == MYOLO_F16 ? 2 : 4, dyes = dy_dtype == MYOLO_F16 ? 2 : 4;
  const TensorView xv{const_cast<unsigned char*>(static_cast<const unsigned char*>(x)) + (size_t)x_coff * xes, B, H, W, xc, x_ctot, x_dtype};
  const TensorView dv{const_cast<unsigned char*>(static_cast<const unsigned char*>(dy)) + (size_t)dy_coff * dyes, B, Ho, Wo, dyc, dy_ctot,
                      dy_dtype};
  const TensorView gv{gin ? static_cast<unsigned char*>(gin) + (size_t)gin_coff * xes : nullptr, B, H, W, xc, gin_ctot, x_dtype};
  cudaStream_t s = (cudaStream_t)stream;
  WeightSlot sl;
  sl.co = co;
  sl.ci = ci;
  sl.k = k;
  sl.set = true;
  sl.w_master = w;
  sl.d_w = dW;
  sl.d_bias = dbias;
  ConvOp dconv;
  int dconv_ready = 0;
  __half* tmp16 = nullptr;
  const size_t need = conv_bwd_tmp16_bytes(xv, dv, co, stride, nullptr);
  if (need) MYOLO_CHECK_CUDA(cudaMalloc(&tmp16, need));
  bool used_side = false;
  rc = conv_backward_views(xv, dv, gin ? &gv : nullptr, sl, k, stride, dil, ConvBwdScratch{tmp16, &dconv, &dconv_ready}, sms,
                           (route & MYOLO_CONV_BWD_SIMT) != 0, (route & MYOLO_CONV_BWD_NO_WGRAD_TC) != 0, s, s, nullptr, &used_side, info);
  const cudaError_t e = cudaStreamSynchronize(s);
  if (tmp16) cudaFree(tmp16);
  if (sl.w_dgrad) cudaFree(sl.w_dgrad);
  if (sl.zero_bias) cudaFree(sl.zero_bias);
  if (sl.dw_packed) cudaFree(sl.dw_packed);
  if (!rc && e != cudaSuccess) {
    set_error("conv_backward: kernel failed: %s", cudaGetErrorString(e));
    rc = MYOLO_E_CUDA;
  }
  return rc;
}

// ------------------------------------------------------------------------------------------------
// gradient exchange: NCCL all-reduce of the flat gradient buffer (nccl_symbol: the libnccl already in the process)
// ------------------------------------------------------------------------------------------------
extern "C" int myolo_allreduce_grads(float* flat_grad, int64_t n, void* nccl_comm, void* stream) {
  NvtxRange nvtx_("myolo_allreduce_grads");
  MYOLO_REQUIRE(flat_grad && n > 0 && nccl_comm, "allreduce_grads: bad arguments");
  return nccl_allreduce_sum(flat_grad, (size_t)n, nccl_comm, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------
// standalone fused conv (per-op parity tests, ncu captures)
// ------------------------------------------------------------------------------------------------
extern "C" int myolo_conv_forward(const void* x, int x_dtype, int B, int H, int W, int x_ctot, int x_coff, void* y, int y_dtype, int y_ctot,
                                  int y_coff, const void* res, int res_ctot, int res_coff, const float* w, int co, int ci, int k, int stride,
                                  int dil, const float* gamma, const float* beta, const float* mean, const float* var, float eps,
                                  const float* bias, int act, int path, int32_t* info, void* stream) {
  NvtxRange nvtx_("myolo_conv_forward");
  MYOLO_REQUIRE(x && y && w && B > 0 && H > 0 && W > 0 && co > 0 && ci > 0 && k >= 1 && k % 2 == 1 && (stride == 1 || stride == 2) &&
                dil >= 1 && path >= 0 && path <= 3, "conv_forward: bad arguments");
  MYOLO_REQUIRE((gamma && beta && mean && var) || (!gamma && !beta && !mean && !var), "conv_forward: partial BN parameters");
  MYOLO_REQUIRE((x_dtype == MYOLO_F16 || x_dtype == MYOLO_F32) && (y_dtype == MYOLO_F16 || y_dtype == MYOLO_F32),
                "conv_forward: x and y must be MYOLO_F16 or MYOLO_F32");
  // the plan's views: x carries ci rounded up to 16 channels (the padding channels hold zeros), y and the residual co
  const int xc = (int)align_up(ci, 16);
  MYOLO_REQUIRE(x_coff >= 0 && x_coff + xc <= x_ctot && y_coff >= 0 && y_coff + co <= y_ctot &&
                (!res || (res_coff >= 0 && res_coff + co <= res_ctot)), "conv_forward: channel slice outside its buffer");
  int sms = 0;
  int rc = check_device(&sms);
  if (rc) return rc;
  const int pad = dil * (k / 2);
  const int Ho = (H + 2 * pad - dil * (k - 1) - 1) / stride + 1, Wo = (W + 2 * pad - dil * (k - 1) - 1) / stride + 1;
  MYOLO_REQUIRE(Ho > 0 && Wo > 0, "conv_forward: empty output map");
  const size_t xes = x_dtype == MYOLO_F16 ? 2 : 4, yes = y_dtype == MYOLO_F16 ? 2 : 4;
  const TensorView xv{const_cast<unsigned char*>(static_cast<const unsigned char*>(x)) + (size_t)x_coff * xes, B, H, W, xc, x_ctot, x_dtype};
  const TensorView yv{static_cast<unsigned char*>(y) + (size_t)y_coff * yes, B, Ho, Wo, co, y_ctot, y_dtype};
  const TensorView rv{const_cast<unsigned char*>(static_cast<const unsigned char*>(res)) + (size_t)res_coff * 2, B, Ho, Wo, co, res_ctot,
                      MYOLO_F16};
  cudaStream_t s = (cudaStream_t)stream;
  WeightSlot sl;
  sl.co = co;
  sl.ci = ci;
  sl.k = k;
  sl.co_pad = conv_n_pad(co);
  sl.ci_pad = xc;
  MYOLO_CHECK_CUDA(cudaMalloc(&sl.w, (size_t)sl.co_pad * k * k * sl.ci_pad * 2));
  MYOLO_CHECK_CUDA(cudaMalloc(&sl.bias, (size_t)sl.co_pad * 4));
  rc = pack_conv_weights(w, co, ci, k, gamma, beta, mean, var, eps, bias, sl.w, sl.bias, sl.co_pad, sl.ci_pad, s);
  ConvOp c;
  if (!rc) rc = conv_forward_views(c, xv, yv, res ? &rv : nullptr, sl, k, stride, dil, act, path == 2, sms);
  if (!rc && (path == 1 || path == 3) && !c.use_tc) {
    set_error("conv_forward: shape not eligible for the tensor-core path");
    rc = MYOLO_E_INVALID;
  }
  if (!rc && path == 3) {      // streamed weights, one A box per tap: the layout the reuse paths are checked against
    c.reuse = false;
    rc = conv_tc_prepare(c, sms);
  }
  if (!rc) rc = c.use_tc ? conv_tc_launch(c, s) : conv_simt_launch(c, s);
  if (!rc && info) conv_info_slots(c, info);
  const cudaError_t e = cudaStreamSynchronize(s);
  cudaFree(sl.w);
  cudaFree(sl.bias);
  if (!rc && e != cudaSuccess) {
    set_error("conv_forward: kernel failed: %s", cudaGetErrorString(e));
    rc = MYOLO_E_CUDA;
  }
  return rc;
}
