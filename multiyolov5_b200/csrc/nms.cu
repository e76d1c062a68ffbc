// utils.general.non_max_suppression (reference utils/general.py:421-509) + torchvision.ops.nms (call site :493) on the device.
//
// Stage 1  (grid over anchors x images): obj>conf filter, conf = cls*obj, best-class (or multi-label) selection, optional
//          class filter; survivors are appended as 64-bit sort keys  (~score_bits << 32 | anchor*nc + cls).
//          The key alone identifies the candidate: boxes/scores are re-read from `pred` later, nothing else is stored.
// Stage 2  (one CTA per image): bitonic sort of the keys (shared memory up to 16384 keys, in-place global otherwise) =
//          descending score with ascending original index as tie break == the stable order torchvision visits boxes in;
//          then greedy suppression in chunks of 256 candidates against the list of already-kept boxes (<= max_det, so the
//          loop stops as soon as 300 boxes are kept: exactly `i[:max_det]` of the reference) with a 256x256 bit matrix
//          for the intra-chunk dependencies.  Every IoU operation is an explicit round-to-nearest fp32 op in the order
//          of the torchvision CPU kernel, so kept indices are bit-exact with the reference.
//
// Apriori labels (myolo_nms_labels, :448-455, the autolabelling of test.py --save-hybrid): image b's k_b label rows [cls, x, y, w, h]
// are virtual rows A .. A + k_b - 1 of that image with box = xywh, obj = 1 and a one-hot class.  Their candidate index i * nc + j
// then sorts after every anchor of the image on equal scores, the position torch.cat((x, v), 0) gives them.  They skip the obj >
// conf_thres pre-filter, as in the reference, and take every later step like any other candidate (so at conf_thres >= 1 they drop out).
#include "common.cuh"

namespace myolo {

static constexpr int kSortSmemKeys = 16384;
static constexpr int kChunk = 256;
static constexpr int kMaxKept = 1024;

struct NmsParams {
  const float* pred;
  int B, A, no, nc;
  float conf_thres, iou_thres, max_wh;
  const int32_t* classes;
  int n_classes, agnostic, multi_label, max_det, max_nms;
  const float* labels;       // [n][5] cls, x, y, w, h (network-input pixels) or nullptr
  const int32_t* label_off;  // [B + 1] image b's rows are labels[label_off[b] .. label_off[b + 1])
  int max_labels;            // bound on any image's label count: the grid and key capacity are sized by it
  int32_t* err;              // MYOLO_NMS_ERR_* bits, OR-ed in
  int32_t* counts;       // [B]
  unsigned long long* keys;  // [B][cap2]
  long cap, cap2;
  float* out;            // [B][max_det][6]
  int32_t* out_count;    // [B]
};

__device__ __forceinline__ bool class_ok(const NmsParams& p, int j) {
  if (p.classes == nullptr) return true;
  for (int k = 0; k < p.n_classes; ++k)
    if (p.classes[k] == j) return true;
  return false;
}

__device__ __forceinline__ void push_key(const NmsParams& p, int b, float score, unsigned idx) {
  const int slot = atomicAdd(&p.counts[b], 1);
  if (slot < p.cap) p.keys[(size_t)b * p.cap2 + slot] = ((unsigned long long)(~__float_as_uint(score)) << 32) | idx;
}

// class score of label row `lab` for class j: the one-hot column times obj = 1 (x[:, 5:] *= x[:, 4:5])
__device__ __forceinline__ float label_score(int lc, int j) { return __fmul_rn(j == lc ? 1.0f : 0.0f, 1.0f); }

__global__ void nms_filter_kernel(NmsParams p) {
  const int b = blockIdx.y;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0 && p.label_off != nullptr && p.label_off[b + 1] - p.label_off[b] > p.max_labels) atomicOr(p.err, MYOLO_NMS_ERR_LABEL_COUNT);
  if (i >= p.A) {
    const int k = i - p.A;
    if (k >= p.max_labels) return;      // also the last block's spare threads, and every thread of myolo_nms (no label table)
    const int k0 = p.label_off[b], nb = p.label_off[b + 1] - k0;
    if (k >= nb) return;
    const float c = p.labels[(size_t)(k0 + k) * 5];
    // l[:, 0].long() must name a class column: ids >= nc are an index error in the reference, and negative ids write 1.0 into a box
    // or obj column (or wrap into the class columns), which is no label at all; both set the error bit here
    if (!(c > -1.0f && c < (float)p.nc)) { atomicOr(p.err, MYOLO_NMS_ERR_LABEL_CLASS); return; }
    const int lc = (int)c;
    if (p.multi_label) {
      for (int j = 0; j < p.nc; ++j) {
        const float s = label_score(lc, j);
        if (s > p.conf_thres && class_ok(p, j)) push_key(p, b, s, (unsigned)((unsigned)i * p.nc + j));
      }
    } else {
      const float s = label_score(lc, lc);        // the one 1.0 is the first maximum
      if (s > p.conf_thres && class_ok(p, lc)) push_key(p, b, s, (unsigned)((unsigned)i * p.nc + lc));
    }
    return;
  }
  const float* row = p.pred + ((size_t)b * p.A + i) * p.no;
  const float obj = row[4];
  if (!(obj > p.conf_thres)) return;                                   // :430,446
  if (p.multi_label) {                                                 // :468-470
    for (int j = 0; j < p.nc; ++j) {
      const float c = __fmul_rn(row[5 + j], obj);                      // :462
      if (c > p.conf_thres && class_ok(p, j)) push_key(p, b, c, (unsigned)(i * p.nc + j));
    }
  } else {                                                             // :471-473 best class, first maximum wins
    float best = __fmul_rn(row[5], obj);
    int bj = 0;
    for (int j = 1; j < p.nc; ++j) {
      const float c = __fmul_rn(row[5 + j], obj);
      if (c > best) { best = c; bj = j; }
    }
    if (best > p.conf_thres && class_ok(p, bj)) push_key(p, b, best, (unsigned)(i * p.nc + bj));
  }
}

template <typename Ptr>
__device__ void bitonic_sort(Ptr keys, int n2) {
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < n2; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = keys[i], c = keys[ixj];
          const bool asc = (i & k) == 0;
          if ((a > c) == asc) { keys[i] = c; keys[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
}

struct Cand { float x1, y1, x2, y2, conf, cls, ox1, oy1, ox2, oy2, area; };

__device__ __forceinline__ Cand load_cand(const NmsParams& p, int b, unsigned long long key) {
  const unsigned idx = (unsigned)(key & 0xffffffffull);
  const unsigned i = idx / (unsigned)p.nc;
  const int j = (int)(idx % (unsigned)p.nc);
  const float* box;
  Cand c;
  if (i >= (unsigned)p.A) {                                                  // a label row: box = xywh, one-hot class, obj 1
    const float* lab = p.labels + (size_t)(p.label_off[b] + (int)(i - (unsigned)p.A)) * 5;
    box = lab + 1;
    c.conf = label_score((int)lab[0], j);
  } else {
    const float* row = p.pred + ((size_t)b * p.A + i) * p.no;
    box = row;
    c.conf = __fmul_rn(row[5 + j], row[4]);
  }
  const float hw = __fdiv_rn(box[2], 2.0f), hh = __fdiv_rn(box[3], 2.0f);   // xywh2xyxy, utils/general.py:265-272
  c.x1 = __fsub_rn(box[0], hw);
  c.y1 = __fsub_rn(box[1], hh);
  c.x2 = __fadd_rn(box[0], hw);
  c.y2 = __fadd_rn(box[1], hh);
  c.cls = (float)j;
  const float off = __fmul_rn(c.cls, p.agnostic ? 0.0f : p.max_wh);          // :491
  c.ox1 = __fadd_rn(c.x1, off);
  c.oy1 = __fadd_rn(c.y1, off);
  c.ox2 = __fadd_rn(c.x2, off);
  c.oy2 = __fadd_rn(c.y2, off);
  c.area = __fmul_rn(__fsub_rn(c.ox2, c.ox1), __fsub_rn(c.oy2, c.oy1));
  return c;
}

// torchvision CPU nms_kernel arithmetic, op for op.  The IEEE division is only executed when the cheap reciprocal estimate is
// within 1e-4 relative of the threshold: everywhere else the comparison result is provably the same, so rows stay bit-exact.
__device__ __forceinline__ bool iou_gt(float ax1, float ay1, float ax2, float ay2, float aarea, float bx1, float by1, float bx2,
                                       float by2, float barea, float thr) {
  const float xx1 = fmaxf(ax1, bx1), yy1 = fmaxf(ay1, by1), xx2 = fminf(ax2, bx2), yy2 = fminf(ay2, by2);
  const float w = fmaxf(0.0f, __fsub_rn(xx2, xx1)), h = fmaxf(0.0f, __fsub_rn(yy2, yy1));
  const float inter = __fmul_rn(w, h);
  const float uni = __fsub_rn(__fadd_rn(aarea, barea), inter);
  const float approx = inter * __frcp_rn(uni);                 // 2 roundings away from the IEEE quotient
  if (approx > thr * 1.0001f) return true;
  if (approx < thr * 0.9999f) return false;
  return __fdiv_rn(inter, uni) > thr;                          // also the path NaN / inf take (never "greater")
}

__global__ void __launch_bounds__(1024) nms_kernel(NmsParams p) {
  extern __shared__ __align__(16) unsigned char nms_smem[];
  unsigned long long* skeys = reinterpret_cast<unsigned long long*>(nms_smem);   // kSortSmemKeys
  float4* kbox = reinterpret_cast<float4*>(nms_smem + (size_t)kSortSmemKeys * 8);  // kMaxKept offset boxes
  float* karea = reinterpret_cast<float*>(kbox + kMaxKept);
  unsigned* mat = reinterpret_cast<unsigned*>(karea + kMaxKept);                 // kChunk x 8 words
  __shared__ int s_nkept, s_alive_words[8];
  __shared__ unsigned s_keepmask[8];
  __shared__ unsigned char s_alive[kChunk];

  const int b = blockIdx.x;
  long n = p.counts[b];
  if (n > p.cap) n = p.cap;
  unsigned long long* gkeys = p.keys + (size_t)b * p.cap2;
  const bool in_smem = n <= kSortSmemKeys;
  int n2 = 1;
  while (n2 < n) n2 <<= 1;
  if (n > 0) {
    if (in_smem) {
      for (int i = threadIdx.x; i < n2; i += blockDim.x) skeys[i] = i < n ? gkeys[i] : ~0ull;
      __syncthreads();
      bitonic_sort(skeys, n2);
    } else {
      for (long i = n + threadIdx.x; i < n2; i += blockDim.x) gkeys[i] = ~0ull;
      __syncthreads();
      bitonic_sort(gkeys, n2);
    }
  }
  if (n > p.max_nms) n = p.max_nms;                                            // :487-488
  if (threadIdx.x == 0) s_nkept = 0;
  __syncthreads();

  const int t = threadIdx.x;
  const int max_det = p.max_det < kMaxKept ? p.max_det : kMaxKept;
  for (long c0 = 0; c0 < n; c0 += kChunk) {
    const int nkept0 = s_nkept;
    if (nkept0 >= max_det) break;
    const int m = (int)((n - c0) < kChunk ? (n - c0) : kChunk);
    Cand me;
    if (t < m) me = load_cand(p, b, in_smem ? skeys[c0 + t] : gkeys[c0 + t]);
    // chunk boxes in shared memory: read by the kept-list check (4 threads per candidate) and by the intra-chunk matrix
    float4* cbox = reinterpret_cast<float4*>(mat + kChunk * 8);
    float* carea = reinterpret_cast<float*>(cbox + kChunk);
    if (t < m) { cbox[t] = make_float4(me.ox1, me.oy1, me.ox2, me.oy2); carea[t] = me.area; }
    __syncthreads();
    {
      // candidate r = t/4 against the kept list: its 4 threads take every fourth kept box (the list reaches max_det = 300 entries)
      const int r = t >> 2, q = t & 3;
      bool dead = false;
      if (r < m) {
        const float4 rb = cbox[r];
        const float ra = carea[r];
        for (int k = q; k < nkept0; k += 4) {
          const float4 kb = kbox[k];
          if (iou_gt(kb.x, kb.y, kb.z, kb.w, karea[k], rb.x, rb.y, rb.z, rb.w, ra, p.iou_thres)) { dead = true; break; }
        }
      }
      unsigned d = dead ? 1u : 0u;
      d |= __shfl_xor_sync(0xffffffffu, d, 1);
      d |= __shfl_xor_sync(0xffffffffu, d, 2);
      if (q == 0) s_alive[r] = (r < m && !d) ? 1 : 0;
    }
    __syncthreads();
    if (t < kChunk) {
      const unsigned bal = __ballot_sync(0xffffffffu, s_alive[t] != 0);
      if ((t & 31) == 0) s_alive_words[t >> 5] = (int)bal;
    }
    __syncthreads();
    {
      // row r = t/4: which later candidates u>r of this chunk would be suppressed by r; the 4 threads of a row take u = r+1+q, +4, ...
      const int r = t >> 2, q = t & 3;
      unsigned wbits[8];
#pragma unroll
      for (int wq = 0; wq < 8; ++wq) wbits[wq] = 0u;
      const bool r_alive = r < m && ((((unsigned)s_alive_words[r >> 5]) >> (r & 31)) & 1u);
      if (r_alive) {
        const float4 rb = cbox[r];
        const float ra = carea[r];
        for (int u = r + 1 + q; u < m; u += 4) {
          const float4 ub = cbox[u];
          if (iou_gt(rb.x, rb.y, rb.z, rb.w, ra, ub.x, ub.y, ub.z, ub.w, carea[u], p.iou_thres)) wbits[u >> 5] |= 1u << (u & 31);
        }
      }
#pragma unroll
      for (int wq = 0; wq < 8; ++wq) {
        unsigned v = wbits[wq];
        v |= __shfl_xor_sync(0xffffffffu, v, 1);
        v |= __shfl_xor_sync(0xffffffffu, v, 2);
        if (q == 0) mat[r * 8 + wq] = v;
      }
    }
    __syncthreads();
    if (t < 32) {
      // serial greedy resolve; lane l (<8) owns word l of the removed mask
      unsigned removed = t < 8 ? ~(unsigned)s_alive_words[t] : 0u;
      unsigned keep = 0u;
      int nk = nkept0;
      for (int i = 0; i < m; ++i) {
        const unsigned wi = __shfl_sync(0xffffffffu, removed, i >> 5);
        const bool kept = !((wi >> (i & 31)) & 1u) && nk < max_det;
        if (kept) {
          if (t < 8) removed |= mat[i * 8 + t];
          if (t == (i >> 5)) keep |= 1u << (i & 31);
          ++nk;
        }
      }
      if (t < 8) s_keepmask[t] = keep;
    }
    __syncthreads();
    if (t < kChunk) {
      // rank of each kept candidate inside the chunk -> position in the kept list / output
      const bool kept = t < m && ((s_keepmask[t >> 5] >> (t & 31)) & 1u);
      int rank = 0;
      for (int wq = 0; wq < (t >> 5); ++wq) rank += __popc(s_keepmask[wq]);
      rank += __popc(s_keepmask[t >> 5] & ((1u << (t & 31)) - 1u));
      if (kept) {
        const int pos = nkept0 + rank;
        kbox[pos] = make_float4(me.ox1, me.oy1, me.ox2, me.oy2);
        karea[pos] = me.area;
        float* o = p.out + ((size_t)b * p.max_det + pos) * 6;
        o[0] = me.x1; o[1] = me.y1; o[2] = me.x2; o[3] = me.y2; o[4] = me.conf; o[5] = me.cls;
      }
    }
    __syncthreads();
    if (t == 0) {
      int tot = 0;
      for (int wq = 0; wq < 8; ++wq) tot += __popc(s_keepmask[wq]);
      s_nkept = nkept0 + tot;
    }
    __syncthreads();
  }
  if (t == 0) p.out_count[b] = s_nkept;
}

}  // namespace myolo

using namespace myolo;

static long next_pow2(long v) {
  long r = 1;
  while (r < v) r <<= 1;
  return r;
}

static long nms_cap(int A, int nc, int multi_label, int max_labels) {
  return multi_label && nc > 1 ? ((long)A + max_labels) * nc : (long)A + max_labels;
}

extern "C" int64_t myolo_nms_workspace_bytes(int B, int A, int no, int multi_label) {
  return 256 + align_up((int64_t)B * 4, 256) + (int64_t)B * next_pow2(nms_cap(A, no - 5, multi_label, 0)) * 8;
}

extern "C" int64_t myolo_nms_labels_workspace_bytes(int B, int A, int no, int multi_label, int max_labels) {
  return 256 + align_up((int64_t)B * 4, 256) + (int64_t)B * next_pow2(nms_cap(A, no - 5, multi_label, max_labels < 0 ? 0 : max_labels)) * 8;
}

static int nms_launch(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes, int n_classes,
                      int agnostic, int multi_label, int max_det, int max_nms, float max_wh, const float* labels, const int32_t* label_off,
                      int max_labels, int32_t* err, float* out, int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream) {
  MYOLO_REQUIRE(pred && out && out_count && workspace, "nms: null pointer");
  MYOLO_REQUIRE(B > 0 && A > 0 && no > 5, "nms: bad shape B=%d A=%d no=%d", B, A, no);
  MYOLO_REQUIRE(max_det > 0 && max_det <= kMaxKept, "nms: max_det must be in [1,%d]", kMaxKept);
  const int nc = no - 5;
  MYOLO_REQUIRE(((long)A + max_labels) * nc < (1l << 32), "nms: (A + max_labels) * nc does not fit the 32-bit candidate index");
  multi_label = multi_label && nc > 1;   // :440
  const long cap = nms_cap(A, nc, multi_label, max_labels);
  MYOLO_REQUIRE(workspace_bytes >= 256 + align_up((int64_t)B * 4, 256) + (int64_t)B * next_pow2(cap) * 8, "nms: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  NmsParams p;
  p.pred = pred; p.B = B; p.A = A; p.no = no; p.nc = nc;
  p.conf_thres = conf_thres; p.iou_thres = iou_thres; p.max_wh = max_wh;
  p.classes = n_classes > 0 ? classes : nullptr; p.n_classes = n_classes;
  p.agnostic = agnostic; p.multi_label = multi_label; p.max_det = max_det; p.max_nms = max_nms;
  p.labels = labels; p.label_off = label_off; p.max_labels = max_labels; p.err = err;
  p.cap = cap;
  p.cap2 = next_pow2(p.cap);
  unsigned char* ws = reinterpret_cast<unsigned char*>(workspace);
  ws = reinterpret_cast<unsigned char*>(align_up((int64_t)ws, 256));
  p.counts = reinterpret_cast<int32_t*>(ws);
  p.keys = reinterpret_cast<unsigned long long*>(ws + align_up((int64_t)B * 4, 256));
  p.out = out; p.out_count = out_count;
  MYOLO_CHECK_CUDA(cudaMemsetAsync(p.counts, 0, (size_t)B * 4, s));
  dim3 g1(ceil_div(A + max_labels, 256), B);
  nms_filter_kernel<<<g1, 256, 0, s>>>(p);
  MYOLO_LAUNCH_CHECK();
  const size_t smem = (size_t)kSortSmemKeys * 8 + kMaxKept * 16 + kMaxKept * 4 + kChunk * 8 * 4 + kChunk * 16 + kChunk * 4;
  static bool attr = false;
  if (!attr) {
    MYOLO_CHECK_CUDA(cudaFuncSetAttribute(nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = true;
  }
  nms_kernel<<<B, 1024, smem, s>>>(p);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_nms(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes,
                         int n_classes, int agnostic, int multi_label, int max_det, int max_nms, float max_wh, float* out,
                         int32_t* out_count, void* workspace, int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_nms");
  return nms_launch(pred, B, A, no, conf_thres, iou_thres, classes, n_classes, agnostic, multi_label, max_det, max_nms, max_wh, nullptr,
                    nullptr, 0, nullptr, out, out_count, workspace, workspace_bytes, stream);
}

extern "C" int myolo_nms_labels(const float* pred, int B, int A, int no, float conf_thres, float iou_thres, const int32_t* classes,
                                int n_classes, int agnostic, int multi_label, int max_det, int max_nms, float max_wh, const float* labels,
                                const int32_t* label_offsets, int max_labels, int32_t* err, float* out, int32_t* out_count, void* workspace,
                                int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_nms_labels");
  MYOLO_REQUIRE(label_offsets && err && max_labels >= 0 && (labels || max_labels == 0), "nms_labels: null pointer or bad max_labels");
  return nms_launch(pred, B, A, no, conf_thres, iou_thres, classes, n_classes, agnostic, multi_label, max_det, max_nms, max_wh,
                    labels, label_offsets, max_labels, err, out, out_count, workspace, workspace_bytes, stream);
}
