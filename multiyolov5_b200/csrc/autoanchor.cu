// Autoanchor (reference utils/autoanchor.py:23-160) on the device: the ratio metric of check_anchors / print_results, and the whole
// genetic evolution of kmean_anchors in one persistent cooperative kernel.  The host keeps the random draws (all gen mutation factors are
// drawn up front in the reference's order: the loop never reads k or the fitness), scipy's k-means and the final writes into Detect.
//
// Exactness (DESIGN.md section 3b): with 1 / anchor_t >= 1/16 every fitness term is 0 or an fp32 value in (1/16, 1], an integer multiple
// of 2^-27; fewer than 2^26 of them sum to an integer below 2^53 times 2^-27, which fp64 holds exactly in any order.  The fitness is that
// sum rounded to fp32 and divided by n in fp32, as torch's CPU mean divides its sum; the result does not depend on the grid.
#include <cooperative_groups.h>

#include "kernels.h"

namespace cg = cooperative_groups;

namespace myolo {

namespace {

constexpr int kThreads = 256;
constexpr int kMetricBlocks = 256;

__device__ __forceinline__ float div_rn(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div_rn(double a, double b) { return __ddiv_rn(a, b); }
__device__ __forceinline__ float rcp_rn(float a) { return __frcp_rn(a); }
__device__ __forceinline__ double rcp_rn(double a) { return __drcp_rn(a); }
__device__ __forceinline__ float cvt_thr(double t, float) { return __double2float_rn(t); }
__device__ __forceinline__ double cvt_thr(double t, double) { return t; }

template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// torch.min(r, 1. / r).min(2)[0] for one label and one anchor: `1. / r` is r.reciprocal() * 1., a correctly rounded reciprocal
template <typename T>
__device__ __forceinline__ T ratio(T w, T h, T kw, T kh) {
  const T r0 = div_rn(w, kw), r1 = div_rn(h, kh);
  return min(min(r0, rcp_rn(r0)), min(r1, rcp_rn(r1)));
}

struct MetricPartial {
  long long n_best, n_x;
  double sum_x, sum_best, sum_x_above;
};

// per block: counts of best > thr and x > thr, and the fp64 sums of x, best and x > thr, in the compute dtype T
template <typename T, typename WT, typename KT>
__global__ void __launch_bounds__(kThreads) anchor_metric_kernel(const WT* __restrict__ wh, long n, const KT* __restrict__ k, int na,
                                                                double thr_d, MetricPartial* __restrict__ part) {
  __shared__ T s_k[2 * MYOLO_ANCHOR_MAX];
  __shared__ MetricPartial s_w[kThreads / 32];
  for (int j = threadIdx.x; j < 2 * na; j += blockDim.x) s_k[j] = (T)k[j];
  __syncthreads();
  const T thr = cvt_thr(thr_d, T(0));
  long long nb = 0, nx = 0;
  double sx = 0.0, sb = 0.0, sxa = 0.0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const T w = (T)wh[2 * i], h = (T)wh[2 * i + 1];
    T best = ratio(w, h, s_k[0], s_k[1]);
    for (int a = 0; a < na; ++a) {
      const T x = ratio(w, h, s_k[2 * a], s_k[2 * a + 1]);
      best = max(best, x);
      sx += (double)x;
      if (x > thr) { ++nx; sxa += (double)x; }
    }
    sb += (double)best;
    nb += best > thr;
  }
  nb = warp_sum(nb); nx = warp_sum(nx); sx = warp_sum(sx); sb = warp_sum(sb); sxa = warp_sum(sxa);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) s_w[warp] = MetricPartial{nb, nx, sx, sb, sxa};
  __syncthreads();
  if (threadIdx.x == 0) {
    MetricPartial p = s_w[0];
    for (int w = 1; w < kThreads / 32; ++w) {
      p.n_best += s_w[w].n_best; p.n_x += s_w[w].n_x;
      p.sum_x += s_w[w].sum_x; p.sum_best += s_w[w].sum_best; p.sum_x_above += s_w[w].sum_x_above;
    }
    part[blockIdx.x] = p;
  }
}

// the blocks' partials in block order (a fixed order: the same sums on every run)
__global__ void anchor_metric_final_kernel(const MetricPartial* __restrict__ part, int n_blocks, myolo_anchor_stats* __restrict__ out) {
  MetricPartial p = part[0];
  for (int b = 1; b < n_blocks; ++b) {
    p.n_best += part[b].n_best; p.n_x += part[b].n_x;
    p.sum_x += part[b].sum_x; p.sum_best += part[b].sum_best; p.sum_x_above += part[b].sum_x_above;
  }
  *out = myolo_anchor_stats{p.n_best, p.n_x, p.sum_x, p.sum_best, p.sum_x_above};
}

template <typename T, typename WT, typename KT>
void launch_metric_t(const void* wh, long n, const void* k, int na, double thr, MetricPartial* part, int grid, cudaStream_t s) {
  anchor_metric_kernel<T, WT, KT><<<grid, kThreads, 0, s>>>(static_cast<const WT*>(wh), n, static_cast<const KT*>(k), na, thr, part);
}

// The evolution.  Generation g = -1 evaluates k0 itself (the reference's initial f = anchor_fitness(k)); generation g >= 0 evaluates
// kg = max(k * v[g], 2.0) and takes it when its fitness is strictly greater.  Each CTA sums its labels' terms, writes the partial to
// partials[g & 1][cta] and meets the others at ONE grid barrier; every CTA then adds all partials (exact, so in any order) and reaches the
// same decision, so no second barrier is needed.  The two partial slots alternate: a CTA writing generation g + 1 cannot overwrite what a
// slower CTA still reads for generation g, because both sit on opposite sides of generation g + 1's barrier.
__global__ void __launch_bounds__(kThreads) anchor_evolve_kernel(const float2* __restrict__ wh, long n, const double* __restrict__ k0, int na,
                                                                const double* __restrict__ v, int gen, float thr, double* partials,
                                                                double* __restrict__ k_out, float* __restrict__ f_out,
                                                                float* __restrict__ fg_out, int* __restrict__ accepted_out) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double s_k[2 * MYOLO_ANCHOR_MAX], s_kg[2 * MYOLO_ANCHOR_MAX];
  __shared__ float s_kf[2 * MYOLO_ANCHOR_MAX];
  __shared__ double s_w[kThreads / 32];
  __shared__ float s_f;
  __shared__ int s_take, s_acc;
  const int m = 2 * na, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int j = threadIdx.x; j < m; j += blockDim.x) s_k[j] = k0[j];
  if (threadIdx.x == 0) { s_f = 0.f; s_acc = 0; }
  const float nf = (float)n;
  for (int g = -1; g < gen; ++g) {
    __syncthreads();
    for (int j = threadIdx.x; j < m; j += blockDim.x) {
      const double kg = g < 0 ? s_k[j] : fmax(__dmul_rn(s_k[j], v[(long)g * m + j]), 2.0);
      s_kg[j] = kg;
      s_kf[j] = __double2float_rn(kg);         // torch.tensor(k, dtype=torch.float32)
    }
    __syncthreads();
    double acc = 0.0;
    for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
      const float2 p = wh[i];
      float best = ratio(p.x, p.y, s_kf[0], s_kf[1]);
      for (int a = 1; a < na; ++a) best = fmaxf(best, ratio(p.x, p.y, s_kf[2 * a], s_kf[2 * a + 1]));
      if (best > thr) acc += (double)best;
    }
    acc = warp_sum(acc);
    if (lane == 0) s_w[warp] = acc;
    __syncthreads();
    double* slot = partials + (g & 1) * (long)gridDim.x;
    if (threadIdx.x == 0) {
      double b = 0.0;
      for (int w = 0; w < kThreads / 32; ++w) b += s_w[w];
      slot[blockIdx.x] = b;
    }
    grid.sync();
    if (warp == 0) {
      double sum = 0.0;
      for (int c = lane; c < (int)gridDim.x; c += 32) sum += __ldcg(slot + c);     // L2: other CTAs wrote it
      sum = warp_sum(sum);
      if (lane == 0) {
        const float fg = __fdiv_rn(__double2float_rn(sum), nf);
        int take = 0;
        if (g < 0) {
          s_f = fg;
          if (blockIdx.x == 0) f_out[0] = fg;
        } else {
          if (blockIdx.x == 0) fg_out[g] = fg;
          take = fg > s_f;
          if (take) { s_f = fg; ++s_acc; }
        }
        s_take = take;
      }
    }
    __syncthreads();
    if (s_take)
      for (int j = threadIdx.x; j < m; j += blockDim.x) s_k[j] = s_kg[j];
  }
  __syncthreads();
  if (blockIdx.x == 0) {
    for (int j = threadIdx.x; j < m; j += blockDim.x) k_out[j] = s_k[j];
    if (threadIdx.x == 0) { f_out[1] = s_f; *accepted_out = s_acc; }
  }
}

int evolve_grid(long n, int* grid) {
  int dev = 0, sms = 0, coop = 0, per_sm = 0;
  MYOLO_CHECK_CUDA(cudaGetDevice(&dev));
  MYOLO_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MYOLO_CHECK_CUDA(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  MYOLO_REQUIRE(coop, "anchor_evolve: the device does not support cooperative launches");
  MYOLO_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, anchor_evolve_kernel, kThreads, 0));
  MYOLO_REQUIRE(per_sm > 0, "anchor_evolve: the kernel cannot be resident");
  *grid = (int)std::max(1L, std::min((long)per_sm * sms, (n + kThreads - 1) / kThreads));
  return 0;
}

}  // namespace

}  // namespace myolo

using namespace myolo;

extern "C" int64_t myolo_anchor_metric_workspace_bytes(void) { return (int64_t)kMetricBlocks * sizeof(MetricPartial); }

extern "C" int myolo_anchor_metric(const void* wh, int wh_dtype, int64_t n, const void* k, int k_dtype, int na, double thr,
                                   myolo_anchor_stats* out, void* workspace, int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_anchor_metric");
  MYOLO_REQUIRE(wh && k && out && workspace && n > 0 && na >= 1 && na <= MYOLO_ANCHOR_MAX, "anchor_metric: bad arguments");
  MYOLO_REQUIRE((wh_dtype == MYOLO_F32 || wh_dtype == MYOLO_F64) && (k_dtype == MYOLO_F32 || k_dtype == MYOLO_F64),
                "anchor_metric: wh and k must be MYOLO_F32 or MYOLO_F64");
  MYOLO_REQUIRE(workspace_bytes >= myolo_anchor_metric_workspace_bytes(), "anchor_metric: workspace too small");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  const int grid = (int)std::max(1L, std::min<long>(kMetricBlocks, (n + kThreads - 1) / kThreads));
  auto* part = static_cast<MetricPartial*>(workspace);
  const bool w64 = wh_dtype == MYOLO_F64, k64 = k_dtype == MYOLO_F64;
  if (!w64 && !k64) launch_metric_t<float, float, float>(wh, n, k, na, thr, part, grid, s);
  else if (!w64 && k64) launch_metric_t<double, float, double>(wh, n, k, na, thr, part, grid, s);
  else if (w64 && !k64) launch_metric_t<double, double, float>(wh, n, k, na, thr, part, grid, s);
  else launch_metric_t<double, double, double>(wh, n, k, na, thr, part, grid, s);
  MYOLO_LAUNCH_CHECK();
  anchor_metric_final_kernel<<<1, 1, 0, s>>>(part, grid, out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t myolo_anchor_evolve_workspace_bytes(int64_t n) {
  int grid = 0;
  if (check_device(nullptr) || n <= 0 || evolve_grid(n, &grid)) return -1;
  return 2 * (int64_t)grid * (int64_t)sizeof(double);
}

extern "C" int myolo_anchor_evolve(const float* wh, int64_t n, const double* k0, int na, const double* v, int gen, double thr,
                                   double* k_out, float* f_out, float* fg_out, int32_t* accepted_out, void* workspace,
                                   int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_anchor_evolve");
  MYOLO_REQUIRE(wh && k0 && k_out && f_out && accepted_out && workspace && na >= 1 && na <= MYOLO_ANCHOR_MAX && gen >= 0 &&
                (gen == 0 || (v && fg_out)), "anchor_evolve: bad arguments");
  // the exact fp64 sum: every term a multiple of 2^-27 in [0, 1] (fp32(thr) >= 1/16) and fewer than 2^26 of them
  MYOLO_REQUIRE(n >= 1 && n < (int64_t(1) << 26), "anchor_evolve: n = %lld labels, needs 1 <= n < 2^26", (long long)n);
  const float thr32 = (float)thr;
  MYOLO_REQUIRE(thr32 >= 0.0625f, "anchor_evolve: 1 / anchor_t = %g, needs anchor_t <= 16", thr);
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  int grid = 0;
  int rc = evolve_grid(n, &grid);
  if (rc) return rc;
  MYOLO_REQUIRE(workspace_bytes >= 2 * (int64_t)grid * (int64_t)sizeof(double), "anchor_evolve: workspace too small");
  double* partials = static_cast<double*>(workspace);
  const float2* wh2 = reinterpret_cast<const float2*>(wh);
  void* args[] = {(void*)&wh2, (void*)&n, (void*)&k0, (void*)&na, (void*)&v, (void*)&gen, (void*)&thr32, (void*)&partials, (void*)&k_out,
                  (void*)&f_out, (void*)&fg_out, (void*)&accepted_out};
  MYOLO_CHECK_CUDA(cudaLaunchCooperativeKernel((const void*)anchor_evolve_kernel, dim3(grid), dim3(kThreads), args, 0, s));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
