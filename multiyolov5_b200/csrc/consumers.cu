// Device-side consumers of the segmentation output (SURVEY.md section 8f rank 2): palette / id look-up (reference detect.py:69-77),
// the visualisation blend cv2.addWeighted(mask, 0.4, im0, 0.6, 0) (detect.py:194) and the validation counters of
// utils/metrics.py:234-275 (pixel accuracy, per-class intersection / prediction / label areas) - each removes a full-resolution
// device->host copy from the reference's loops.  Integer / byte work: bit exact.  HBM bound, one pass each.
#include "kernels.h"

namespace myolo {

__device__ __forceinline__ int load_cls(const void* p, int dtype, long i) {
  return dtype == MYOLO_U8 ? (int)reinterpret_cast<const unsigned char*>(p)[i] : (int)reinterpret_cast<const long long*>(p)[i];
}

// out[i][c] = lut[idx[i]][reverse ? ch-1-c : c];  optional blend: dst[i][c] = sat(rint(out*alpha + im[i][c]*beta))  (fp32, round half even)
__global__ void lut_blend_kernel(const void* idx, int idx_dtype, long n, const unsigned char* __restrict__ lut, int n_entries, int ch,
                                 int reverse, unsigned char* out, const unsigned char* im, float alpha, float beta, unsigned char* blend) {
  extern __shared__ unsigned char s_lut[];
  for (int k = threadIdx.x; k < n_entries * ch; k += blockDim.x) s_lut[k] = lut[k];
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
  }
}

int launch_lut_blend(const void* idx, int idx_dtype, long n, const unsigned char* lut, int n_entries, int ch, int reverse, unsigned char* out,
                     const unsigned char* im, float alpha, float beta, unsigned char* blend, cudaStream_t s) {
  MYOLO_REQUIRE(idx && lut && n > 0 && n_entries > 0 && ch > 0 && n_entries * ch <= 4096 && (out || blend) && (!blend || im),
                "lut_blend: bad arguments");
  MYOLO_REQUIRE(idx_dtype == MYOLO_U8 || idx_dtype == MYOLO_I64, "lut_blend: class map must be uint8 or int64");
  lut_blend_kernel<<<(int)std::min<long>(132L * 8, (n + 255) / 256), 256, n_entries * ch, s>>>(idx, idx_dtype, n, lut, n_entries, ch, reverse, out,
                                                                                              im, alpha, beta, blend);
  MYOLO_LAUNCH_CHECK();
  return 0;
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

int launch_seg_hist(const void* pred, int pred_dtype, const long long* target, long n, int n_cls, unsigned long long* counters,
                    cudaStream_t s) {
  MYOLO_REQUIRE(pred && target && counters && n > 0 && n_cls > 0 && n_cls <= 1024, "seg_hist: bad arguments");
  MYOLO_REQUIRE(pred_dtype == MYOLO_U8 || pred_dtype == MYOLO_I64, "seg_hist: prediction must be uint8 or int64");
  // one block sees at most 2^32 - 1 pixels per counter: blocks of <= 2^24 pixels each
  const int blocks = (int)std::max<long>(std::min<long>(132L * 8, (n + 255) / 256), (n + (1L << 24) - 1) >> 24);
  seg_hist_kernel<<<blocks, 256, (2 + 3 * n_cls) * sizeof(unsigned int), s>>>(pred, pred_dtype, target, n, n_cls, counters);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo
