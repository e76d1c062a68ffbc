// --image-weights on the device (reference train.py:255,305-316, utils/general.py:216-240), bit for bit with numpy and Python's random:
//   class weights  labels_to_class_weights: exact per-class label counts, empty bins -> 1, w = 1 / count, w / (numpy's sum of w)
//   image weights  labels_to_image_weights: per image the histogram of its labels' classes, (cw * count) summed over nc as numpy sums it
//   weighted draw  random.choices(range(n), weights=iw, k=n) from n host-drawn random() values: sequential cumulative sums
//                  (itertools.accumulate), total = cum[-1] + 0.0, then bisect_right(cum, u * total, 0, n - 1) per draw
// numpy's sum over a contiguous axis of m <= MYOLO_IW_NC_MAX values (DESIGN.md section 3c): the pairwise sum of all m values (below 8: a
// sequential sum from -0.0; up to 128: 8 strided accumulators combined as ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the rest in order;
// above: split at n2 = m/2 - (m/2)%8), added to the reduction's initial 0.0.  fp64 is written with __dadd_rn / __dmul_rn / __ddiv_rn so
// that nvcc cannot contract any of it into fused multiply-adds.
#include <math_constants.h>

#include "kernels.h"

namespace myolo {

namespace {

constexpr int kLeaf = 128;              // numpy's PW_BLOCKSIZE
constexpr int kDepth = 4;               // the pairwise recursion's depth for m <= 1024
static_assert(MYOLO_IW_NC_MAX <= 1024, "kDepth covers m <= 1024");
constexpr int kHistThreads = 256;
constexpr int kImageWarps = 8;
constexpr int kScanThreads = 1024;
constexpr int kScanChunk = 4096;        // fp64 values staged in shared memory per step of the scan
constexpr int kDrawThreads = 256;

template <class T>
__device__ double pairwise_leaf(const T& term, int s, int m) {
  if (m < 8) {
    double res = -0.0;
    for (int i = 0; i < m; ++i) res = __dadd_rn(res, term(s + i));
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = term(s + j);
  int i = 8;
  for (; i < m - (m % 8); i += 8)
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], term(s + i + j));
  double res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
  for (; i < m; ++i) res = __dadd_rn(res, term(s + i));
  return res;
}

template <int D, class T>
__device__ double pairwise(const T& term, int s, int m) {
  if constexpr (D == 0) {
    return pairwise_leaf(term, s, m);
  } else {
    if (m <= kLeaf) return pairwise_leaf(term, s, m);
    int h = m / 2;
    h -= h % 8;
    return __dadd_rn(pairwise<D - 1>(term, s, h), pairwise<D - 1>(term, s + h, m - h));
  }
}

// np.add.reduce over m contiguous values: the pairwise sum added to the initial 0.0
template <class T>
__device__ double numpy_sum(const T& term, int m) {
  return __dadd_rn(0.0, pairwise<kDepth>(term, 0, m));
}

// astype(int) of a float32 class: truncation toward zero; anything outside [0, nc) (NaN included) is -1
__device__ __forceinline__ int class_of(float v, int nc) {
  return (v > -1.0f && v < (float)nc) ? (int)v : -1;
}

__global__ void __launch_bounds__(kHistThreads) class_count_kernel(const float* __restrict__ cls, long long n_labels, int nc,
                                                                 unsigned long long* __restrict__ counts, int* __restrict__ status) {
  extern __shared__ unsigned int s_hist[];
  for (int c = threadIdx.x; c < nc; c += blockDim.x) s_hist[c] = 0;
  __syncthreads();
  bool bad = false;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_labels; i += (long long)gridDim.x * blockDim.x) {
    const int c = class_of(cls[i], nc);
    if (c < 0) bad = true;
    else atomicAdd(&s_hist[c], 1u);
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(status, MYOLO_IW_BAD_CLASS);
  for (int c = threadIdx.x; c < nc; c += blockDim.x)
    if (s_hist[c]) atomicAdd(counts + c, (unsigned long long)s_hist[c]);
}

__global__ void __launch_bounds__(kHistThreads) class_weights_kernel(const unsigned long long* __restrict__ counts, int nc,
                                                                   double* __restrict__ weights) {
  __shared__ double s_w[MYOLO_IW_NC_MAX];
  __shared__ double s_sum;
  for (int c = threadIdx.x; c < nc; c += blockDim.x) {
    const unsigned long long k = counts[c];
    s_w[c] = __ddiv_rn(1.0, (double)(k ? k : 1ull));       // weights[weights == 0] = 1; weights = 1 / weights
  }
  __syncthreads();
  if (threadIdx.x == 0) s_sum = numpy_sum([&](int c) { return s_w[c]; }, nc);
  __syncthreads();
  for (int c = threadIdx.x; c < nc; c += blockDim.x) weights[c] = __ddiv_rn(s_w[c], s_sum);
}

// one warp per image: its histogram in shared memory, then lane 0 sums cw * count over nc in numpy's order
__global__ void __launch_bounds__(kImageWarps * 32) image_weights_kernel(const float* __restrict__ cls, const long long* __restrict__ offsets,
                                                                         long long n, const double* __restrict__ cw, int nc,
                                                                         double* __restrict__ iw, int* __restrict__ status) {
  extern __shared__ double s_cw[];                                 // nc fp64, then one nc-entry histogram per warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned int* hist = reinterpret_cast<unsigned int*>(s_cw + nc) + warp * nc;
  for (int c = threadIdx.x; c < nc; c += blockDim.x) s_cw[c] = cw[c];
  __syncthreads();
  bool bad = false;
  for (long long i = blockIdx.x * (long long)kImageWarps + warp; i < n; i += (long long)gridDim.x * kImageWarps) {
    for (int c = lane; c < nc; c += 32) hist[c] = 0;
    __syncwarp();
    const long long b = offsets[i], e = offsets[i + 1];
    for (long long j = b + lane; j < e; j += 32) {
      const int c = class_of(cls[j], nc);
      if (c < 0) bad = true;
      else atomicAdd(&hist[c], 1u);
    }
    __syncwarp();
    if (lane == 0) iw[i] = numpy_sum([&](int c) { return __dmul_rn(s_cw[c], (double)hist[c]); }, nc);
    __syncwarp();
  }
  if (__any_sync(0xffffffffu, bad) && lane == 0) atomicOr(status, MYOLO_IW_BAD_CLASS);
}

// itertools.accumulate(w) by one thread, staged through shared memory in chunks; then random.choices' checks on the total
__global__ void __launch_bounds__(kScanThreads, 1) weighted_scan_kernel(const double* __restrict__ w, long long n, double* __restrict__ cum,
                                                                       double* __restrict__ total, int* __restrict__ status) {
  __shared__ double s[kScanChunk];
  double run = -0.0;                                               // -0.0 + w[0] == w[0]: accumulate's first element as is
  for (long long base = 0; base < n; base += kScanChunk) {
    const int m = (int)min((long long)kScanChunk, n - base);
    for (int i = threadIdx.x; i < m; i += blockDim.x) s[i] = w[base + i];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll 8
      for (int i = 0; i < m; ++i) {
        run = __dadd_rn(run, s[i]);
        s[i] = run;
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) cum[base + i] = s[i];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double t = __dadd_rn(run, 0.0);                           // total = cum_weights[-1] + 0.0
    *total = t;
    if (t <= 0.0) atomicOr(status, MYOLO_IW_TOTAL_NONPOS);
    else if (!isfinite(t)) atomicOr(status, MYOLO_IW_TOTAL_NONFINITE);
  }
}

// bisect_right(cum, u[i] * total, 0, n - 1)
__global__ void __launch_bounds__(kDrawThreads) weighted_draw_kernel(const double* __restrict__ cum, const double* __restrict__ total,
                                                                     const double* __restrict__ u, long long n, int* __restrict__ idx,
                                                                     const int* __restrict__ status) {
  if (*status & (MYOLO_IW_TOTAL_NONPOS | MYOLO_IW_TOTAL_NONFINITE)) return;
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double x = __dmul_rn(u[i], *total);
  long long lo = 0, hi = n - 1;
  while (lo < hi) {
    const long long mid = (lo + hi) / 2;
    if (x < cum[mid]) hi = mid;
    else lo = mid + 1;
  }
  idx[i] = (int)lo;
}

int sm_count() {
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms > 0 ? sms : 1;
}

}  // namespace

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_class_weights(const float* cls, int64_t n_labels, int nc, int64_t* counts, double* weights, int32_t* status,
                                   void* stream) {
  NvtxRange nvtx_("myolo_class_weights");
  MYOLO_REQUIRE((cls || n_labels == 0) && n_labels >= 0 && counts && weights && status, "class_weights: bad arguments");
  MYOLO_REQUIRE(nc >= 1 && nc <= MYOLO_IW_NC_MAX, "class_weights: nc = %d, needs 1 <= nc <= %d", nc, MYOLO_IW_NC_MAX);
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_CHECK_CUDA(cudaMemsetAsync(counts, 0, sizeof(unsigned long long) * nc, s));
  const long long want = (n_labels + kHistThreads - 1) / kHistThreads;
  const int grid = (int)max(1LL, min(want, (long long)sm_count() * 8));
  class_count_kernel<<<grid, kHistThreads, sizeof(unsigned int) * nc, s>>>(cls, n_labels, nc, reinterpret_cast<unsigned long long*>(counts),
                                                                           status);
  MYOLO_LAUNCH_CHECK();
  class_weights_kernel<<<1, kHistThreads, 0, s>>>(reinterpret_cast<unsigned long long*>(counts), nc, weights);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_image_weights(const float* cls, const int64_t* offsets, int64_t n, const double* cw, int nc, double* iw,
                                   int32_t* status, void* stream) {
  NvtxRange nvtx_("myolo_image_weights");
  MYOLO_REQUIRE(cls && offsets && cw && iw && status && n >= 1, "image_weights: bad arguments");
  MYOLO_REQUIRE(nc >= 1 && nc <= MYOLO_IW_NC_MAX, "image_weights: nc = %d, needs 1 <= nc <= %d", nc, MYOLO_IW_NC_MAX);
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  const size_t smem = sizeof(double) * nc + sizeof(unsigned int) * nc * kImageWarps;
  const long long want = (n + kImageWarps - 1) / kImageWarps;
  const int grid = (int)max(1LL, min(want, (long long)sm_count() * 16));
  image_weights_kernel<<<grid, kImageWarps * 32, smem, s>>>(cls, reinterpret_cast<const long long*>(offsets), n, cw, nc, iw, status);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_weighted_draw(const double* w, const double* u, int64_t n, double* cum, double* total, int32_t* idx, int32_t* status,
                                   void* stream) {
  NvtxRange nvtx_("myolo_weighted_draw");
  MYOLO_REQUIRE(w && u && cum && total && idx && status, "weighted_draw: bad arguments");
  MYOLO_REQUIRE(n >= 1 && n < (int64_t(1) << 31), "weighted_draw: n = %lld, needs 1 <= n < 2^31", (long long)n);
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  weighted_scan_kernel<<<1, kScanThreads, 0, s>>>(w, n, cum, total, status);
  MYOLO_LAUNCH_CHECK();
  weighted_draw_kernel<<<(unsigned)((n + kDrawThreads - 1) / kDrawThreads), kDrawThreads, 0, s>>>(cum, total, u, n, idx, status);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
