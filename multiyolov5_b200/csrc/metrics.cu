// Detection validation statistics (reference test.py:175,183-265 and utils/metrics.py:24-112), bit exact with the reference's fp32 /
// float64 arithmetic on the CPU.
//
//   det_match_kernel   one CTA per image: targets to native-space boxes, predictions scaled and clipped, box_iou, the best target of
//                      the prediction's class, the greedy assignment in NMS row order -> one stats-store slot per (image, row)
//   ap_* kernels       ap_per_class over the whole store: compaction, a stable LSD radix sort on (class, descending conf), then one
//                      CTA per (class, IoU column) for the cumulative sums, the precision envelope, np.interp and np.trapz
//
// Ordering of tied confidences: the reference sorts with np.argsort(-conf), which is not stable, so its result for two predictions
// of one class with the same conf and different `correct` rows depends on the machine.  Ours is defined as stable in (image, row)
// order; it equals the reference whenever tied predictions of one class have identical `correct` rows.
//
// All float / double arithmetic uses explicit _rn intrinsics so that nvcc cannot contract it into fused multiply-adds.
#include "kernels.h"

namespace myolo {

constexpr int kMatchThreads = 256;
constexpr int kMaxLabels = 1024;        // targets per image
constexpr int kMaxDetRows = 1024;       // NMS rows per image
constexpr int kSortWarps = 8;           // warps per sort block; each warp owns one contiguous segment
constexpr int kMaxSegments = 512;
constexpr int kApThreads = 512;

__device__ __forceinline__ float scale_x(float v, float pad, float gain, float hi) {
  return fminf(fmaxf(__fdiv_rn(__fsub_rn(v, pad), gain), 0.f), hi);
}

// test.py:175,223-224: a target [x, y, w, h] (normalised) to pixels, xywh2xyxy, scale_coords(ratio_pad) and clip_coords
__device__ __forceinline__ float4 target_box(const float* t, float H, float W, float padw, float padh, float gain, float w0, float h0) {
  const float x = __fmul_rn(t[0], W), y = __fmul_rn(t[1], H), bw = __fmul_rn(t[2], W), bh = __fmul_rn(t[3], H);
  const float hw = __fdiv_rn(bw, 2.f), hh = __fdiv_rn(bh, 2.f);
  float4 bx;
  bx.x = scale_x(__fsub_rn(x, hw), padw, gain, w0);
  bx.y = scale_x(__fsub_rn(y, hh), padh, gain, h0);
  bx.z = scale_x(__fadd_rn(x, hw), padw, gain, w0);
  bx.w = scale_x(__fadd_rn(y, hh), padh, gain, h0);
  return bx;
}

__device__ __forceinline__ float box_area(float4 b) { return __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y)); }

// general.box_iou of one pair in either operand order (min / max and area1 + area2 commute)
__device__ __forceinline__ float pair_iou(float4 a, float aa, float4 t, float ta) {
  const float iw = fmaxf(__fsub_rn(fminf(a.z, t.z), fmaxf(a.x, t.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(a.w, t.w), fmaxf(a.y, t.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(aa, ta), inter));
}

// torch.max over a row: the first NaN if any, else the first maximum
__device__ __forceinline__ void take_max(float v, int k, bool& have, float& best, int& bi) {
  if (!have) { have = true; best = v; bi = k; return; }
  if (isnan(best)) return;
  if (isnan(v) || v > best) { best = v; bi = k; }
}

__global__ void __launch_bounds__(kMatchThreads) det_match_kernel(
    const float* __restrict__ dets, const int32_t* __restrict__ counts, int max_det, const float* __restrict__ targets, int n_targets,
    float H, float W, const float* __restrict__ geom, const float* __restrict__ iouv, int img_base, uint16_t* st_correct, float* st_conf,
    uint8_t* st_cls, int32_t* st_rows, unsigned long long* tcount, int32_t* err) {
  __shared__ float4 s_tbox[kMaxLabels];
  __shared__ float s_tarea[kMaxLabels];
  __shared__ float s_tcls[kMaxLabels];
  __shared__ unsigned char s_taken[kMaxLabels];
  __shared__ float s_best[kMaxDetRows];
  __shared__ short s_bidx[kMaxDetRows];
  __shared__ uint16_t s_bits[kMaxDetRows];
  __shared__ int s_wcount[kMatchThreads / 32];
  __shared__ int s_nl;
  __shared__ float s_iouv[10];
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* g = geom + 5 * b;
  const float h0 = g[0], w0 = g[1], gain = g[2], padw = g[3], padh = g[4];
  if (tid < 10) s_iouv[tid] = iouv[tid];
  if (tid == 0) s_nl = 0;
  __syncthreads();

  // this image's targets, in row order (targets[:, 0] == si): stable compaction by warp ballots
  const float fb = (float)b;
  for (int base = 0; base < n_targets; base += kMatchThreads) {
    const int i = base + tid;
    const bool mine = i < n_targets && targets[(long)i * 6] == fb;
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) s_wcount[warp] = __popc(m);
    __syncthreads();
    int off = s_nl;
    for (int w = 0; w < warp; ++w) off += s_wcount[w];
    if (mine) {
      const int k = off + __popc(m & ((1u << lane) - 1u));
      const float* t = targets + (long)i * 6;
      if (k >= kMaxLabels) {
        atomicOr(err, MYOLO_DET_ERR_LABELS);
      } else {
        const float c = t[1];
        if (!(c >= 0.f && c < 256.f && c == floorf(c))) {
          atomicOr(err, MYOLO_DET_ERR_TARGET_CLASS);
          s_tcls[k] = -1.f;                               // matches no prediction
        } else {
          s_tcls[k] = c;
          atomicAdd(&tcount[(int)c], 1ull);
        }
        // targets[:, 2:] *= [w, h, w, h]; xywh2xyxy; scale_coords(ratio_pad); clip_coords
        const float4 bx = target_box(t + 2, H, W, padw, padh, gain, w0, h0);
        s_tbox[k] = bx;
        s_tarea[k] = box_area(bx);
        s_taken[k] = 0;
      }
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < kMatchThreads / 32; ++w) tot += s_wcount[w];
      s_nl += tot;
    }
    __syncthreads();
  }
  const int nl = min(s_nl, kMaxLabels);
  const int n = min(max(counts[b], 0), max_det);
  const long slot0 = (long)(img_base + b) * max_det;

  // each prediction's best target among the targets of its class (box_iou(...).max(1))
  for (int p = tid; p < n; p += kMatchThreads) {
    const float* r = dets + ((long)b * max_det + p) * 6;
    const float pc = r[5];
    if (!(pc >= 0.f && pc < 256.f && pc == floorf(pc))) atomicOr(err, MYOLO_DET_ERR_PRED_CLASS);
    const float4 pb = make_float4(scale_x(r[0], padw, gain, w0), scale_x(r[1], padh, gain, h0), scale_x(r[2], padw, gain, w0),
                                  scale_x(r[3], padh, gain, h0));
    const float a1 = box_area(pb);
    bool have = false;
    float best = 0.f;
    int bi = -1;
    for (int k = 0; k < nl; ++k) {
      if (s_tcls[k] != pc) continue;
      take_max(pair_iou(pb, a1, s_tbox[k], s_tarea[k]), k, have, best, bi);
    }
    uint16_t bits = 0;
    if (have)
      for (int j = 0; j < 10; ++j) bits |= (uint16_t)(best > s_iouv[j]) << j;
    s_best[p] = have ? best : __int_as_float(0x7fc00000);     // no target of its class: never matches
    s_bidx[p] = (short)bi;
    s_bits[p] = bits;
  }
  __syncthreads();

  // greedy assignment in NMS row order: a prediction takes its best target only if that target is still free
  if (tid == 0) {
    for (int p = 0; p < n; ++p) {
      uint16_t c = 0;
      if (s_best[p] > s_iouv[0] && !s_taken[s_bidx[p]]) {
        s_taken[s_bidx[p]] = 1;
        c = s_bits[p];
      }
      s_bits[p] = c;
    }
    st_rows[img_base + b] = n;
  }
  __syncthreads();
  for (int p = tid; p < n; p += kMatchThreads) {
    const float* r = dets + ((long)b * max_det + p) * 6;
    st_correct[slot0 + p] = s_bits[p];
    st_conf[slot0 + p] = r[4];
    const float pc = r[5];
    st_cls[slot0 + p] = (pc >= 0.f && pc < 256.f) ? (uint8_t)pc : (uint8_t)255;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------------
// ConfusionMatrix.process_batch (the fork's utils/metrics.py:115-162), one CTA per image
//
// The fork keeps the pairs with IoU > iou_thres, sorts them by IoU (descending) and keeps each detection's first pair, sorts again and
// keeps each label's first pair: every detection keeps its best label, then every label its best detection among those that kept it.
// numpy's argsort there is not stable, so exact IoU ties are not pinned by the fork; here a detection's tie goes to the lower label
// index and a label's tie to the lower detection row (the filtered detections keep their row order).
// ---------------------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool class_in(float c, int nc) { return c >= 0.f && c < (float)nc && c == floorf(c); }

__global__ void __launch_bounds__(kMatchThreads) confusion_kernel(
    const float* __restrict__ dets, const int32_t* __restrict__ counts, int max_det, const float* __restrict__ targets, int n_targets,
    float H, float W, const float* __restrict__ geom, int nc, float conf_thres, float iou_thres, int require_rows,
    unsigned long long* matrix, int32_t* err) {
  __shared__ float4 s_tbox[kMaxLabels];
  __shared__ float s_tarea[kMaxLabels];
  __shared__ short s_tcls[kMaxLabels];      // -1: class outside [0, nc)
  __shared__ short s_lmatch[kMaxLabels];    // the label's detection row, -1 none
  __shared__ short s_dlab[kMaxDetRows];     // the detection's best label, -1 none (or dropped by conf)
  __shared__ float s_diou[kMaxDetRows];
  __shared__ short s_dcls[kMaxDetRows];
  __shared__ unsigned char s_dmatched[kMaxDetRows];
  __shared__ int s_wcount[kMatchThreads / 32];
  __shared__ int s_nl, s_any;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float h0 = 0.f, w0 = 0.f, gain = 1.f, padw = 0.f, padh = 0.f;
  if (geom) { h0 = geom[5 * b]; w0 = geom[5 * b + 1]; gain = geom[5 * b + 2]; padw = geom[5 * b + 3]; padh = geom[5 * b + 4]; }
  if (tid == 0) { s_nl = 0; s_any = 0; }
  __syncthreads();

  // this image's labels in row order, as det_match_kernel gathers them
  const float fb = (float)b;
  for (int base = 0; base < n_targets; base += kMatchThreads) {
    const int i = base + tid;
    const bool mine = i < n_targets && targets[(long)i * 6] == fb;
    const unsigned m = __ballot_sync(0xffffffffu, mine);
    if (lane == 0) s_wcount[warp] = __popc(m);
    __syncthreads();
    int off = s_nl;
    for (int w = 0; w < warp; ++w) off += s_wcount[w];
    if (mine) {
      const int k = off + __popc(m & ((1u << lane) - 1u));
      const float* t = targets + (long)i * 6;
      if (k >= kMaxLabels) {
        atomicOr(err, MYOLO_DET_ERR_LABELS);
      } else {
        const bool ok = class_in(t[1], nc);
        if (!ok) atomicOr(err, MYOLO_DET_ERR_TARGET_CLASS);
        s_tcls[k] = ok ? (short)t[1] : (short)-1;
        const float4 bx = geom ? target_box(t + 2, H, W, padw, padh, gain, w0, h0) : make_float4(t[2], t[3], t[4], t[5]);
        s_tbox[k] = bx;
        s_tarea[k] = box_area(bx);
        s_lmatch[k] = -1;
      }
    }
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int w = 0; w < kMatchThreads / 32; ++w) tot += s_wcount[w];
      s_nl += tot;
    }
    __syncthreads();
  }
  const int nl = min(s_nl, kMaxLabels);
  const int n = min(max(counts[b], 0), max_det);
  if (require_rows && (nl == 0 || n == 0)) return;         // test.py:189-192: no process_batch for this image

  // detections = detections[detections[:, 4] > conf]; each detection's best label with IoU > iou_thres
  for (int p = tid; p < n; p += kMatchThreads) {
    const float* r = dets + ((long)b * max_det + p) * 6;
    const bool active = r[4] > conf_thres;
    short dc = -1;
    if (active) {
      if (class_in(r[5], nc)) dc = (short)r[5];
      else atomicOr(err, MYOLO_DET_ERR_PRED_CLASS);
    }
    int bk = -1;
    float best = 0.f;
    if (active) {
      const float4 pb = geom ? make_float4(scale_x(r[0], padw, gain, w0), scale_x(r[1], padh, gain, h0), scale_x(r[2], padw, gain, w0),
                                           scale_x(r[3], padh, gain, h0))
                             : make_float4(r[0], r[1], r[2], r[3]);
      const float pa = box_area(pb);
      for (int k = 0; k < nl; ++k) {
        const float iou = pair_iou(s_tbox[k], s_tarea[k], pb, pa);
        if (iou > iou_thres && (bk < 0 || iou > best)) { best = iou; bk = k; }
      }
    }
    s_dlab[p] = (short)bk;
    s_diou[p] = best;
    s_dcls[p] = dc;
    s_dmatched[p] = 0;
  }
  __syncthreads();
  // each label's best detection among those whose best label it is
  for (int k = tid; k < nl; k += kMatchThreads) {
    int bp = -1;
    float best = 0.f;
    for (int p = 0; p < n; ++p)
      if (s_dlab[p] == k && (bp < 0 || s_diou[p] > best)) { best = s_diou[p]; bp = p; }
    s_lmatch[k] = (short)bp;
    if (bp >= 0) { s_dmatched[bp] = 1; s_any = 1; }
  }
  __syncthreads();
  const unsigned long long ld = (unsigned long long)nc + 1;
  for (int k = tid; k < nl; k += kMatchThreads) {
    const int gc = s_tcls[k], bp = s_lmatch[k];
    if (gc < 0) continue;
    if (bp >= 0) {
      if (s_dcls[bp] >= 0) atomicAdd(&matrix[gc * ld + s_dcls[bp]], 1ull);      // correct
    } else {
      atomicAdd(&matrix[nc * ld + gc], 1ull);                                     // background FP
    }
  }
  if (s_any)                                                                      // `if n:` — only when the image has a match
    for (int p = tid; p < n; p += kMatchThreads)
      if (dets[((long)b * max_det + p) * 6 + 4] > conf_thres && !s_dmatched[p] && s_dcls[p] >= 0)
        atomicAdd(&matrix[s_dcls[p] * ld + nc], 1ull);                            // background FN
}

// ---------------------------------------------------------------------------------------------------------------------------------
// ap_per_class
// ---------------------------------------------------------------------------------------------------------------------------------
struct ApWorkspace {
  int32_t* img_off;        // n_images exclusive prefix of the row counts
  int32_t* hdr;            // [0] any correct bit, [1] N, [2..8) unused, [8..8+256) predictions per class
  unsigned long long* keys[2];
  uint32_t* vals[2];       // store slot index
  int32_t* digit;          // 256 * S
  int32_t* tpc;            // ncol * Nmax
  double* env;             // ncol * Nmax
};

static size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

static int sort_segments(long nmax, long* seg_len) {
  long L = std::max<long>(1024, (nmax + kMaxSegments - 1) / kMaxSegments);
  L = (L + 31) & ~31L;
  *seg_len = L;
  int S = (int)((nmax + L - 1) / L);
  return ((std::max(S, 1) + kSortWarps - 1) / kSortWarps) * kSortWarps;
}

static size_t ap_layout(int n_images, int max_det, int ncol, ApWorkspace* w, char* base) {
  const long nmax = (long)n_images * max_det;
  long L;
  const int S = sort_segments(nmax, &L);
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = base ? base + off : nullptr; off += align256(bytes); return p; };
  ApWorkspace t;
  t.img_off = (int32_t*)take(sizeof(int32_t) * n_images);
  t.hdr = (int32_t*)take(sizeof(int32_t) * (8 + 256));
  t.keys[0] = (unsigned long long*)take(sizeof(unsigned long long) * nmax);
  t.keys[1] = (unsigned long long*)take(sizeof(unsigned long long) * nmax);
  t.vals[0] = (uint32_t*)take(sizeof(uint32_t) * nmax);
  t.vals[1] = (uint32_t*)take(sizeof(uint32_t) * nmax);
  t.digit = (int32_t*)take(sizeof(int32_t) * 256 * (size_t)S);
  t.tpc = (int32_t*)take(sizeof(int32_t) * (size_t)ncol * nmax);
  t.env = (double*)take(sizeof(double) * (size_t)ncol * nmax);
  if (w) *w = t;
  return off;
}

// block-wide inclusive scan (sum or max) over kApThreads values in shared memory
template <typename T, bool kMax>
__device__ T block_scan(T v, T* sh) {
  const int tid = threadIdx.x;
  sh[tid] = v;
  __syncthreads();
  for (int d = 1; d < (int)blockDim.x; d <<= 1) {
    T o = tid >= d ? sh[tid - d] : T(0);
    __syncthreads();
    if (tid >= d) sh[tid] = kMax ? (o > sh[tid] ? o : sh[tid]) : sh[tid] + o;
    __syncthreads();
  }
  T r = sh[tid];
  __syncthreads();
  return r;
}

__global__ void __launch_bounds__(1024) ap_offsets_kernel(const int32_t* __restrict__ rows, int n_images, int max_det, int32_t* img_off,
                                                          int32_t* hdr) {
  __shared__ int sh[1024];
  __shared__ int carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n_images; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < n_images ? min(max(rows[i], 0), max_det) : 0;
    const int inc = block_scan<int, false>(v, sh);
    if (i < n_images) img_off[i] = carry + inc - v;
    __syncthreads();
    if (threadIdx.x == blockDim.x - 1) carry += inc;
    __syncthreads();
  }
  if (threadIdx.x == 0) hdr[1] = carry;
}

__device__ __forceinline__ unsigned long long sort_key(uint8_t cls, float conf) {
  uint32_t u = __float_as_uint(conf);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);     // ascending order of conf
  return ((unsigned long long)cls << 32) | (unsigned long long)(~u);   // class ascending, conf descending
}

__global__ void ap_compact_kernel(const uint16_t* __restrict__ correct, const float* __restrict__ conf, const uint8_t* __restrict__ cls,
                                  const int32_t* __restrict__ rows, int max_det, uint16_t colmask, const int32_t* __restrict__ img_off,
                                  int32_t* hdr, unsigned long long* keys, uint32_t* vals) {
  const int img = blockIdx.x;
  const int r = blockIdx.y * blockDim.x + threadIdx.x;
  const int n = min(max(rows[img], 0), max_det);
  if (r >= n) return;
  const long slot = (long)img * max_det + r;
  const int pos = img_off[img] + r;
  keys[pos] = sort_key(cls[slot], conf[slot]);
  vals[pos] = (uint32_t)slot;
  atomicAdd(&hdr[8 + cls[slot]], 1);
  if (correct[slot] & colmask) hdr[0] = 1;
}

__global__ void __launch_bounds__(kSortWarps * 32) radix_hist_kernel(const unsigned long long* __restrict__ keys, const int32_t* hdr,
                                                                     long seg_len, int S, int shift, int32_t* digit) {
  __shared__ int sh[kSortWarps][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int k = lane; k < 256; k += 32) sh[warp][k] = 0;
  __syncwarp();
  const long N = hdr[1];
  const int seg = blockIdx.x * kSortWarps + warp;
  const long start = seg * seg_len, end = min(N, start + seg_len);
  for (long i = start + lane; i < end; i += 32) atomicAdd(&sh[warp][(int)(keys[i] >> shift) & 255], 1);
  __syncwarp();
  for (int k = lane; k < 256; k += 32) digit[(long)k * S + seg] = sh[warp][k];
}

__global__ void __launch_bounds__(1024) radix_scan_kernel(int32_t* digit, long n) {
  __shared__ int sh[1024];
  const long chunk = (n + blockDim.x - 1) / blockDim.x;
  const long a = threadIdx.x * chunk, e = min(n, a + chunk);
  int sum = 0;
  for (long i = a; i < e; ++i) sum += digit[i];
  const int inc = block_scan<int, false>(sum, sh);
  int run = inc - sum;
  for (long i = a; i < e; ++i) {
    const int v = digit[i];
    digit[i] = run;
    run += v;
  }
}

__global__ void __launch_bounds__(kSortWarps * 32) radix_scatter_kernel(const unsigned long long* __restrict__ kin,
                                                                        const uint32_t* __restrict__ vin, const int32_t* hdr, long seg_len,
                                                                        int S, int shift, const int32_t* __restrict__ digit,
                                                                        unsigned long long* kout, uint32_t* vout) {
  __shared__ int base[kSortWarps][256];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int seg = blockIdx.x * kSortWarps + warp;
  for (int k = lane; k < 256; k += 32) base[warp][k] = digit[(long)k * S + seg];
  __syncwarp();
  const long N = hdr[1];
  const long start = seg * seg_len, end = min(N, start + seg_len);
  for (long r = start; r < end; r += 32) {       // rounds of 32 keys in order: stable within the segment
    const long i = r + lane;
    const bool valid = i < end;
    unsigned long long k = 0;
    uint32_t v = 0;
    int d = 256 + lane;                            // invalid lanes match nobody
    if (valid) {
      k = kin[i];
      v = vin[i];
      d = (int)(k >> shift) & 255;
    }
    const unsigned m = __match_any_sync(0xffffffffu, d);
    const int rank = __popc(m & ((1u << lane) - 1u));
    int pos = 0;
    if (valid) pos = base[warp][d] + rank;
    __syncwarp();
    if (valid && lane == __ffs(m) - 1) base[warp][d] += __popc(m);
    __syncwarp();
    if (valid) {
      kout[pos] = k;
      vout[pos] = v;
    }
  }
}

// recall / precision / -conf of the class segment, by sorted index k
struct ApSeg {
  const uint32_t* slots;
  const int32_t* tpc;
  const double* env;
  const float* conf;
  int n;
  double nl;        // n_l + 1e-16
};

__device__ __forceinline__ double seg_recall(const ApSeg& s, int k) { return __ddiv_rn((double)s.tpc[k], s.nl); }
__device__ __forceinline__ double seg_precision(const ApSeg& s, int k) { return __ddiv_rn((double)s.tpc[k], (double)(k + 1)); }
__device__ __forceinline__ double seg_negconf(const ApSeg& s, int k) { return -(double)s.conf[s.slots[k]]; }

// np.interp value from index j = (#xp <= x) - 1 of a curve with `len` points
__device__ __forceinline__ double interp_at(double x, int j, int len, double left, double xj, double xj1, double fj, double fj1) {
  if (j < 0) return left;
  if (j == len - 1 || xj == x) return fj;
  const double slope = __ddiv_rn(__dsub_rn(fj1, fj), __dsub_rn(xj1, xj));
  return __dadd_rn(__dmul_rn(slope, __dsub_rn(x, xj)), fj);
}

__global__ void __launch_bounds__(kApThreads) ap_class_kernel(const uint16_t* __restrict__ correct, const float* __restrict__ conf,
                                                              const unsigned long long* __restrict__ tcount, const int32_t* __restrict__ hdr,
                                                              const uint32_t* __restrict__ sorted, long nmax, int ncol,
                                                              const double* __restrict__ px, const double* __restrict__ x101,
                                                              int32_t* tpc_ws, double* env_ws, double* out_ap, double* out_p, double* out_r) {
  __shared__ double sh_d[kApThreads];
  __shared__ int sh_i[kApThreads];
  __shared__ double s_y[101];
  const int c = blockIdx.x, col = blockIdx.y, tid = threadIdx.x;
  const unsigned long long nl = tcount[c];
  if (nl == 0) return;
  int row = 0, start = 0;
  for (int k = 0; k < c; ++k) {
    row += tcount[k] > 0;
    start += hdr[8 + k];
  }
  const int n = hdr[8 + c];
  if (n == 0) {                                    // no predictions of a labelled class: zero rows (utils/metrics.py:54-55)
    if (tid == 0) out_ap[(long)row * ncol + col] = 0.0;
    if (col == 0)
      for (int t = tid; t < 1000; t += blockDim.x) out_p[(long)row * 1000 + t] = out_r[(long)row * 1000 + t] = 0.0;
    return;
  }
  ApSeg s;
  s.slots = sorted + start;
  s.tpc = tpc_ws + (long)col * nmax + start;
  s.env = env_ws + (long)col * nmax + start;
  s.conf = conf;
  s.n = n;
  s.nl = __dadd_rn((double)nl, 1e-16);
  int32_t* tpc = tpc_ws + (long)col * nmax + start;
  double* env = env_ws + (long)col * nmax + start;

  // tpc = tp.cumsum(0): per-thread contiguous chunks + one block scan
  const int chunk = (n + blockDim.x - 1) / blockDim.x;
  const int a = min(n, tid * chunk), e = min(n, a + chunk);
  int cnt = 0;
  for (int k = a; k < e; ++k) cnt += (correct[s.slots[k]] >> col) & 1;
  int run = block_scan<int, false>(cnt, sh_i) - cnt;
  double cmax = 0.0;
  for (int k = a; k < e; ++k) {
    run += (correct[s.slots[k]] >> col) & 1;
    tpc[k] = run;
    const double p = __ddiv_rn((double)run, (double)(k + 1));
    cmax = p > cmax ? p : cmax;
  }
  // precision envelope (suffix max): a max scan over the chunk maxima in reversed thread order
  const int rt = blockDim.x - 1 - tid;
  sh_d[tid] = cmax;
  __syncthreads();
  const double rev = sh_d[rt];
  __syncthreads();
  sh_d[tid] = block_scan<double, true>(rev, sh_d);              // max over the chunks of threads >= blockDim-1-tid
  __syncthreads();
  double later = rt > 0 ? sh_d[rt - 1] : 0.0;                   // max over the chunks after this thread's
  __syncthreads();
  for (int k = e - 1; k >= a; --k) {
    const double p = __ddiv_rn((double)tpc[k], (double)(k + 1));
    later = p > later ? p : later;
    env[k] = later;
  }
  __syncthreads();

  // compute_ap: mrec = [0, recall..., recall[-1] + 0.01], envelope of [1, precision..., 0]; np.interp at 101 points
  if (tid < 101) {
    const double x = x101[tid];
    int lo = 0, hi = n;                            // first k with recall(k) > x
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (seg_recall(s, mid) <= x) lo = mid + 1; else hi = mid;
    }
    const double rlast = seg_recall(s, n - 1);
    const double mlast = __dadd_rn(rlast, 0.01);
    const int j = lo + (mlast <= x ? 1 : 0);       // (#mrec <= x) - 1, with mrec[0] = 0 <= x
    const int len = n + 2;
    auto mrec = [&](int m) { return m == 0 ? 0.0 : (m <= n ? seg_recall(s, m - 1) : mlast); };
    auto mpre = [&](int m) { return m == 0 ? 1.0 : (m <= n ? s.env[m - 1] : 0.0); };
    double y;
    if (j >= len - 1) y = 0.0;
    else y = interp_at(x, j, len, 0.0, mrec(j), mrec(j + 1), mpre(j), mpre(j + 1));
    s_y[tid] = y;
  }
  __syncthreads();
  if (tid == 0) {                                  // np.trapz: d * (y[1:] + y[:-1]) / 2.0 summed in numpy's pairwise order (100 terms)
    double r[8];
    auto term = [&](int i) { return __ddiv_rn(__dmul_rn(__dsub_rn(x101[i + 1], x101[i]), __dadd_rn(s_y[i + 1], s_y[i])), 2.0); };
    for (int k = 0; k < 8; ++k) r[k] = term(k);
    for (int i = 8; i < 96; i += 8)
      for (int k = 0; k < 8; ++k) r[k] = __dadd_rn(r[k], term(i + k));
    double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
    for (int i = 96; i < 100; ++i) res = __dadd_rn(res, term(i));
    out_ap[(long)row * ncol + col] = __dadd_rn(0.0, res);
  }
  if (col != 0) return;
  // the p / r curves at IoU 0.5: np.interp(-px, -conf, recall | precision, left=0 | 1)
  for (int t = tid; t < 1000; t += blockDim.x) {
    const double x = -px[t];
    int lo = 0, hi = n;                            // first k with -conf(k) > x
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (seg_negconf(s, mid) <= x) lo = mid + 1; else hi = mid;
    }
    const int j = lo - 1;
    double xj = 0.0, xj1 = 0.0, rj = 0.0, rj1 = 0.0, pj = 0.0, pj1 = 0.0;
    if (j >= 0) {
      xj = seg_negconf(s, j);
      rj = seg_recall(s, j);
      pj = seg_precision(s, j);
      if (j + 1 < n) {
        xj1 = seg_negconf(s, j + 1);
        rj1 = seg_recall(s, j + 1);
        pj1 = seg_precision(s, j + 1);
      }
    }
    out_r[(long)row * 1000 + t] = interp_at(x, j, n, 0.0, xj, xj1, rj, rj1);
    out_p[(long)row * 1000 + t] = interp_at(x, j, n, 1.0, xj, xj1, pj, pj1);
  }
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_det_match(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets, int H, int W,
                               const float* geom, const float* iouv, int img_base, uint16_t* st_correct, float* st_conf, uint8_t* st_cls,
                               int32_t* st_rows, uint64_t* tcount, int32_t* err, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(dets && counts && geom && iouv && st_correct && st_conf && st_cls && st_rows && tcount && err, "det_match: null argument");
  MYOLO_REQUIRE(B > 0 && max_det > 0 && max_det <= kMaxDetRows && H > 0 && W > 0 && img_base >= 0 && n_targets >= 0 &&
                (n_targets == 0 || targets), "det_match: bad arguments (max_det <= %d)", kMaxDetRows);
  det_match_kernel<<<B, kMatchThreads, 0, s>>>(dets, counts, max_det, targets, n_targets, (float)H, (float)W, geom, iouv, img_base,
                                               st_correct, st_conf, st_cls, st_rows, reinterpret_cast<unsigned long long*>(tcount), err);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_confusion_update(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets,
                                      int H, int W, const float* geom, int nc, float conf_thres, float iou_thres, int require_rows,
                                      int64_t* matrix, int32_t* err, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(dets && counts && matrix && err, "confusion: null argument");
  MYOLO_REQUIRE(B > 0 && max_det > 0 && max_det <= kMaxDetRows && nc > 0 && nc <= 4096 && n_targets >= 0 && (n_targets == 0 || targets) &&
                (geom == nullptr || (H > 0 && W > 0)), "confusion: bad arguments (max_det <= %d, nc <= 4096)", kMaxDetRows);
  confusion_kernel<<<B, kMatchThreads, 0, s>>>(dets, counts, max_det, targets, n_targets, (float)H, (float)W, geom, nc, conf_thres, iou_thres,
                                               require_rows, reinterpret_cast<unsigned long long*>(matrix), err);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t myolo_det_ap_workspace_bytes(int n_images, int max_det, int ncol) {
  if (n_images <= 0 || max_det <= 0 || ncol <= 0) return 0;
  return (int64_t)ap_layout(n_images, max_det, ncol, nullptr, nullptr);
}

extern "C" int myolo_det_ap(const uint16_t* correct, const float* conf, const uint8_t* cls, const int32_t* rows, int n_images, int max_det,
                            int ncol, const uint64_t* tcount, const double* px, const double* x101, double* out_ap, double* out_p,
                            double* out_r, int32_t* out_info, void* workspace, int64_t workspace_bytes, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(correct && conf && cls && rows && tcount && px && x101 && out_ap && out_p && out_r && out_info && workspace,
                "det_ap: null argument");
  MYOLO_REQUIRE(n_images > 0 && max_det > 0 && ncol >= 1 && ncol <= 16, "det_ap: bad arguments");
  const long nmax = (long)n_images * max_det;
  MYOLO_REQUIRE(nmax < (1L << 31), "det_ap: store too large");
  MYOLO_REQUIRE(workspace_bytes >= myolo_det_ap_workspace_bytes(n_images, max_det, ncol), "det_ap: workspace too small");
  ApWorkspace w;
  ap_layout(n_images, max_det, ncol, &w, (char*)workspace);
  long L;
  const int S = sort_segments(nmax, &L);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(w.hdr, 0, sizeof(int32_t) * (8 + 256), s));
  ap_offsets_kernel<<<1, 1024, 0, s>>>(rows, n_images, max_det, w.img_off, w.hdr);
  MYOLO_LAUNCH_CHECK();
  ap_compact_kernel<<<dim3(n_images, (max_det + 255) / 256), 256, 0, s>>>(correct, conf, cls, rows, max_det, (uint16_t)((1u << ncol) - 1u),
                                                                          w.img_off, w.hdr, w.keys[0], w.vals[0]);
  MYOLO_LAUNCH_CHECK();
  int cur = 0;
  for (int shift = 0; shift < 40; shift += 8) {
    radix_hist_kernel<<<S / kSortWarps, kSortWarps * 32, 0, s>>>(w.keys[cur], w.hdr, L, S, shift, w.digit);
    MYOLO_LAUNCH_CHECK();
    radix_scan_kernel<<<1, 1024, 0, s>>>(w.digit, 256L * S);
    MYOLO_LAUNCH_CHECK();
    radix_scatter_kernel<<<S / kSortWarps, kSortWarps * 32, 0, s>>>(w.keys[cur], w.vals[cur], w.hdr, L, S, shift, w.digit, w.keys[cur ^ 1],
                                                                    w.vals[cur ^ 1]);
    MYOLO_LAUNCH_CHECK();
    cur ^= 1;
  }
  ap_class_kernel<<<dim3(256, ncol), kApThreads, 0, s>>>(correct, conf, reinterpret_cast<const unsigned long long*>(tcount), w.hdr, w.vals[cur],
                                                         nmax, ncol, px, x101, w.tpc, w.env, out_ap, out_p, out_r);
  MYOLO_LAUNCH_CHECK();
  MYOLO_CHECK_CUDA(cudaMemcpyAsync(out_info, w.hdr, 2 * sizeof(int32_t), cudaMemcpyDeviceToDevice, s));
  return 0;
}
