// Device-side consumers of the segmentation output (SURVEY.md section 8f rank 2): palette / id look-up (reference detect.py:69-77),
// the visualisation blend cv2.addWeighted(mask, 0.4, im0, 0.6, 0) (detect.py:194) and the validation counters of
// utils/metrics.py:234-275 (pixel accuracy, per-class intersection / prediction / label areas) - each removes a full-resolution
// device->host copy from the reference's loops.  Integer / byte work: bit exact.  HBM bound, one pass each.
#include "kernels.h"

namespace myolo {

__device__ __forceinline__ int load_cls(const void* p, int dtype, long i) {
  return dtype == MYOLO_U8 ? (int)reinterpret_cast<const unsigned char*>(p)[i] : (int)reinterpret_cast<const long long*>(p)[i];
}

// out[i][c] = lut[idx[i]][reverse ? ch-1-c : c];  optional blend: dst[i][c] = sat(rint(out*alpha + im[i][c]*beta))  (fp32, round half even);
// optional second table: out2[i][c] = lut2[idx[i]][c] (same entries, ch2 channels, its own order), from the same class-map read
__global__ void lut_blend_kernel(const void* idx, int idx_dtype, long n, const unsigned char* __restrict__ lut, int n_entries, int ch,
                                 int reverse, unsigned char* out, const unsigned char* im, float alpha, float beta, unsigned char* blend,
                                 const unsigned char* __restrict__ lut2, int ch2, unsigned char* out2) {
  extern __shared__ unsigned char s_lut[];
  unsigned char* s_lut2 = s_lut + n_entries * ch;
  for (int k = threadIdx.x; k < n_entries * ch; k += blockDim.x) s_lut[k] = lut[k];
  if (out2)
    for (int k = threadIdx.x; k < n_entries * ch2; k += blockDim.x) s_lut2[k] = lut2[k];
  __syncthreads();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    int v = load_cls(idx, idx_dtype, i);
    v = min(max(v, 0), n_entries - 1);
    for (int c = 0; c < ch; ++c) {
      const unsigned char m = s_lut[v * ch + (reverse ? ch - 1 - c : c)];
      if (out) out[i * ch + c] = m;
      if (blend) {
        const float r = __fadd_rn(__fmul_rn((float)m, alpha), __fmul_rn((float)im[i * ch + c], beta));
        blend[i * ch + c] = (unsigned char)min(max(__float2int_rn(r), 0), 255);
      }
    }
    if (out2)
      for (int c = 0; c < ch2; ++c) out2[i * ch2 + c] = s_lut2[v * ch2 + c];
  }
}

// detect.py:166-177 over a batch of padded NMS rows, one CTA per frame.  geom[b] = {pad_x, pad_y, gain, w0, h0}, each already rounded to
// fp32 as torch's CPU kernels round a Python scalar.  In place on rows [0, counts[b]): x -= pad, x /= gain, clamp to the frame, round half to
// even (scale_coords(...).round(), fp32 IEEE like the reference's CPU run).  xywhn (nullable): (xyxy2xywh(xyxy) / gn) of the rounded box.
// class_counts (nullable): (B, nc) rows per integral class id in [0, nc).
__global__ void detect_boxes_kernel(float* rows, const int32_t* counts, int max_det, const float* geom, int nc, float* xywhn,
                                    int32_t* class_counts) {
  extern __shared__ int s_cnt[];
  const int b = blockIdx.x;
  const float px = geom[b * 5 + 0], py = geom[b * 5 + 1], gain = geom[b * 5 + 2], w0 = geom[b * 5 + 3], h0 = geom[b * 5 + 4];
  if (class_counts)
    for (int k = threadIdx.x; k < nc; k += blockDim.x) s_cnt[k] = 0;
  __syncthreads();
  const int n = min(max(counts[b], 0), max_det);
  for (int r = threadIdx.x; r < n; r += blockDim.x) {
    float* row = rows + ((long)b * max_det + r) * 6;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float lim = (j & 1) ? h0 : w0;
      const float x = __fdiv_rn(__fsub_rn(row[j], (j & 1) ? py : px), gain);
      v[j] = rintf(fminf(fmaxf(x, 0.f), lim));
      row[j] = v[j];
    }
    if (xywhn) {
      float* o = xywhn + ((long)b * max_det + r) * 4;
      o[0] = __fdiv_rn(__fmul_rn(__fadd_rn(v[0], v[2]), 0.5f), w0);
      o[1] = __fdiv_rn(__fmul_rn(__fadd_rn(v[1], v[3]), 0.5f), h0);
      o[2] = __fdiv_rn(__fsub_rn(v[2], v[0]), w0);
      o[3] = __fdiv_rn(__fsub_rn(v[3], v[1]), h0);
    }
    if (class_counts) {
      const float c = row[5];
      if (c >= 0.f && c < (float)nc && c == truncf(c)) atomicAdd(&s_cnt[(int)c], 1);
    }
  }
  if (class_counts) {
    __syncthreads();
    for (int k = threadIdx.x; k < nc; k += blockDim.x) class_counts[(long)b * nc + k] = s_cnt[k];
  }
}

// autoShape's scale_coords(shape1, y[:, :4], shape0) (reference models/common.py:668-669), one CTA per image: as detect_boxes_kernel
// without the round, then Detections.__init__'s xyxy2xywh and its divisions by gn = (w0, h0, w0, h0, 1, 1) (models/common.py:680-688)
__global__ void scale_boxes_kernel(float* rows, const int32_t* counts, int max_det, const float* geom, float* xywh, float* xyxyn,
                                   float* xywhn) {
  const int b = blockIdx.x;
  const float px = geom[b * 5 + 0], py = geom[b * 5 + 1], gain = geom[b * 5 + 2], w0 = geom[b * 5 + 3], h0 = geom[b * 5 + 4];
  const float gn[6] = {w0, h0, w0, h0, 1.f, 1.f};
  const int n = min(max(counts[b], 0), max_det);
  for (int r = threadIdx.x; r < n; r += blockDim.x) {
    const long o = ((long)b * max_det + r) * 6;
    float a[6], w[6];
#pragma unroll
    for (int j = 0; j < 6; ++j) a[j] = rows[o + j];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x = __fdiv_rn(__fsub_rn(a[j], (j & 1) ? py : px), gain);
      a[j] = fminf(fmaxf(x, 0.f), (j & 1) ? h0 : w0);
      rows[o + j] = a[j];
    }
    w[0] = __fdiv_rn(__fadd_rn(a[0], a[2]), 2.f);
    w[1] = __fdiv_rn(__fadd_rn(a[1], a[3]), 2.f);
    w[2] = __fsub_rn(a[2], a[0]);
    w[3] = __fsub_rn(a[3], a[1]);
    w[4] = a[4];
    w[5] = a[5];
#pragma unroll
    for (int j = 0; j < 6; ++j) {
      if (xywh) xywh[o + j] = w[j];
      if (xyxyn) xyxyn[o + j] = __fdiv_rn(a[j], gn[j]);
      if (xywhn) xywhn[o + j] = __fdiv_rn(w[j], gn[j]);
    }
  }
}

// counters[0] = correct, [1] = labeled, [2..2+n) intersection, [2+n..2+2n) prediction area, [2+2n..2+3n) label area  (accumulated)
__global__ void seg_hist_kernel(const void* pred, int pred_dtype, const long long* __restrict__ target, long n, int n_cls,
                                unsigned long long* counters) {
  extern __shared__ unsigned int sh[];     // 2 + 3*n_cls block-local counters
  const int nc = 2 + 3 * n_cls;
  for (int k = threadIdx.x; k < nc; k += blockDim.x) sh[k] = 0;
  __syncthreads();
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = target[i];
    if (t < 0) continue;                                  // ignore label (-1): removed from prediction, label and intersection areas
    const int p = load_cls(pred, pred_dtype, i);
    atomicAdd(&sh[1], 1u);
    if (p >= 0 && p < n_cls) atomicAdd(&sh[2 + n_cls + p], 1u);
    if (t < n_cls) atomicAdd(&sh[2 + 2 * n_cls + (int)t], 1u);
    if (p == t) {
      atomicAdd(&sh[0], 1u);
      if (p < n_cls) atomicAdd(&sh[2 + p], 1u);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < nc; k += blockDim.x)
    if (sh[k]) atomicAdd(&counters[k], (unsigned long long)sh[k]);
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_seg_lut_blend(const void* idx, int idx_dtype, int64_t n, const uint8_t* lut, int n_entries, int ch, int reverse,
                                   uint8_t* out, const uint8_t* im, float alpha, float beta, uint8_t* blend, const uint8_t* lut2, int ch2,
                                   uint8_t* out2, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(idx && lut && n > 0 && n_entries > 0 && ch > 0 && n_entries * ch <= 4096 && (out || blend || out2) && (!blend || im),
                "lut_blend: bad arguments");
  MYOLO_REQUIRE(!out2 || (lut2 && ch2 > 0 && n_entries * ch2 <= 4096), "lut_blend: the second table needs lut2 and 0 < channels2");
  MYOLO_REQUIRE(idx_dtype == MYOLO_U8 || idx_dtype == MYOLO_I64, "lut_blend: class map must be uint8 or int64");
  const int smem = n_entries * (ch + (out2 ? ch2 : 0));
  lut_blend_kernel<<<(int)std::min<long>(132L * 8, (n + 255) / 256), 256, smem, s>>>(idx, idx_dtype, n, lut, n_entries, ch, reverse, out, im,
                                                                                     alpha, beta, blend, lut2, out2 ? ch2 : 0, out2);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_detect_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, int nc, float* xywhn,
                                  int32_t* class_counts, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(rows && counts && geom && B > 0 && max_det > 0, "detect_boxes: bad arguments");
  MYOLO_REQUIRE(!class_counts || (nc > 0 && nc <= 4096), "detect_boxes: class counts need 0 < nc <= 4096");
  detect_boxes_kernel<<<B, 128, class_counts ? nc * (int)sizeof(int) : 0, s>>>(rows, counts, max_det, geom, nc, xywhn, class_counts);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_scale_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, float* xywh, float* xyxyn,
                                 float* xywhn, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(rows && counts && geom && B > 0 && max_det > 0, "scale_boxes: bad arguments");
  scale_boxes_kernel<<<B, 128, 0, s>>>(rows, counts, max_det, geom, xywh, xyxyn, xywhn);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_seg_metrics(const void* pred, int pred_dtype, const int64_t* target, int64_t n, int n_cls, uint64_t* counters,
                                 void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(pred && target && counters && n > 0 && n_cls > 0 && n_cls <= 1024, "seg_hist: bad arguments");
  MYOLO_REQUIRE(pred_dtype == MYOLO_U8 || pred_dtype == MYOLO_I64, "seg_hist: prediction must be uint8 or int64");
  // one block sees at most 2^32 - 1 pixels per counter: blocks of <= 2^24 pixels each
  const int blocks = (int)std::max<long>(std::min<long>(132L * 8, (n + 255) / 256), (n + (1L << 24) - 1) >> 24);
  seg_hist_kernel<<<blocks, 256, (2 + 3 * n_cls) * sizeof(unsigned int), s>>>(pred, pred_dtype, reinterpret_cast<const long long*>(target), n,
                                                                              n_cls, reinterpret_cast<unsigned long long*>(counters));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
