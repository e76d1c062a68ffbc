// scipy.cluster.vq.kmeans(obs, k, iter, thresh) for an int k and d = 2 (kmean_anchors' `kmeans(wh / s, n, iter=30)`, reference
// utils/autoanchor.py:125) on the device, bit for bit with scipy: one CTA runs one restart from its host-drawn start, every restart in one
// ordinary launch.  The rules (DESIGN.md section 3b):
//   vq        dist2 = (c0 - x0)^2 + (c1 - x1)^2 rounded op by op (no FMA), first code with the smallest dist2, sqrt correctly rounded
//   mean      numpy's pairwise sum of the distances: leaves of <= 128 from its recursion, each summed as numpy does (8 accumulators), the
//             partials combined along the recursion's own tree; then / n
//   means     per cluster the sequential fp64 sum in observation order (scipy's update_cluster_means) / member count; empty clusters
//             dropped, the survivors renumbered in order
//   loop      while |prev - cur| > thresh from prev = inf; then one more vq with the final book gives the restart's distortion
//   best      the first restart with dist < best (strict, from inf), picked by the last CTA to finish
#include <math_constants.h>

#include "kernels.h"

namespace myolo {

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kLeaf = 128;              // numpy's PW_BLOCKSIZE
constexpr int kDepth = 40;              // the recursion's depth for n < 2^31 is below 27
static_assert(kWarps >= MYOLO_KMEANS_KMAX, "one warp per cluster");

__host__ __device__ __forceinline__ long long split(long long m) {    // numpy's n2 = n / 2; n2 -= n2 % 8
  const long long h = m / 2;
  return h - h % 8;
}

long long count_leaves(long long m) { return m <= kLeaf ? 1 : count_leaves(split(m)) + count_leaves(m - split(m)); }

struct Layout {
  long long leaves, stride, starts_off, part_off, codes_off;
};

Layout layout(long long n) {
  Layout l;
  l.leaves = count_leaves(n);
  l.starts_off = 0;                                                         // int32 leaf starts, leaves + 1
  l.part_off = (l.starts_off + 4 * (l.leaves + 1) + 15) / 16 * 16;          // fp64 leaf partials
  l.codes_off = l.part_off + 8 * l.leaves;                                  // uint8 codes, n
  l.stride = (l.codes_off + n + 255) / 256 * 256;
  return l;
}
constexpr long long kHeader = 256;      // the done counter

// the leaves' starts in order, by a depth-first walk of numpy's recursion from n
__device__ void enumerate_leaves(int n, int* starts) {
  int size[kDepth], from[kDepth];
  unsigned char right[kDepth];
  int top = 0, leaf = 0;
  size[0] = n; from[0] = 0; right[0] = 0;
  for (;;) {
    while (size[top] > kLeaf) {                 // descend to the leftmost leaf
      size[top + 1] = (int)split(size[top]); from[top + 1] = from[top]; right[top + 1] = 0;
      ++top;
    }
    starts[leaf++] = from[top];
    while (top > 0 && right[top]) --top;        // climb past finished right children
    if (top == 0) break;
    const int h = (int)split(size[top - 1]);    // go to the right sibling
    size[top] = size[top - 1] - h; from[top] = from[top - 1] + h; right[top] = 1;
  }
  starts[leaf] = n;
}

// numpy's pairwise sum of the leaf partials: left + right at every node of its recursion
__device__ double tree_sum(int n, const double* part) {
  int size[kDepth];
  double left[kDepth];
  unsigned char right[kDepth];
  int top = 0, leaf = 0;
  size[0] = n; right[0] = 0;
  for (;;) {
    while (size[top] > kLeaf) {
      size[top + 1] = (int)split(size[top]); right[top + 1] = 0;
      ++top;
    }
    double v = part[leaf++];
    for (;;) {
      if (top == 0) return v;
      if (!right[top]) break;
      v = __dadd_rn(left[top - 1], v);          // a right child finished: its parent's sum
      --top;
    }
    left[top - 1] = v;                          // a left child finished: keep it, go to the right sibling
    size[top] = size[top - 1] - (int)split(size[top - 1]); right[top] = 1;
  }
}

// one observation's code and distance (rule 2), the code written to workspace
__device__ __forceinline__ double nearest(const double2* __restrict__ obs, int i, const double2* book, int kc,
                                          unsigned char* __restrict__ code) {
  const double2 x = obs[i];
  double best = CUDART_INF;
  int bc = 0;
  for (int j = 0; j < kc; ++j) {
    const double a = __dsub_rn(book[j].x, x.x), b = __dsub_rn(book[j].y, x.y);
    const double d2 = __dadd_rn(__dmul_rn(a, a), __dmul_rn(b, b));
    if (d2 < best) { best = d2; bc = j; }
  }
  code[i] = (unsigned char)bc;
  return __dsqrt_rn(best);
}

// vq over every leaf, one leaf per thread in turn; each leaf's partial as numpy's pairwise_sum forms it
__device__ void vq_leaves(const double2* __restrict__ obs, const int* __restrict__ starts, int n_leaves, const double2* book, int kc,
                          unsigned char* __restrict__ code, double* __restrict__ part) {
  for (int l = threadIdx.x; l < n_leaves; l += blockDim.x) {
    const int s = starts[l], m = starts[l + 1] - s;
    double res;
    if (m < 8) {
      res = 0.0;
      for (int i = 0; i < m; ++i) res = __dadd_rn(res, nearest(obs, s + i, book, kc, code));
    } else {
      double r[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) r[j] = nearest(obs, s + j, book, kc, code);
      int i = 8;
      for (; i < m - (m % 8); i += 8)
#pragma unroll
        for (int j = 0; j < 8; ++j) r[j] = __dadd_rn(r[j], nearest(obs, s + i + j, book, kc, code));
      res = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), __dadd_rn(r[2], r[3])), __dadd_rn(__dadd_rn(r[4], r[5]), __dadd_rn(r[6], r[7])));
      for (; i < m; ++i) res = __dadd_rn(res, nearest(obs, s + i, book, kc, code));
    }
    part[l] = res;
  }
}

// cluster c's member sums in observation order (lane 0: feature 0, lane 1: feature 1) and its member count, by one warp
__device__ void cluster_sum(const double2* __restrict__ obs, const unsigned char* __restrict__ code, int n, int c, int lane, double2* sum,
                            int* count) {
  double acc = 0.0;
  int cnt = 0;
  for (int base = 0; base < n; base += 32) {
    const int i = base + lane;
    const bool hit = i < n && code[i] == c;
    unsigned m = __ballot_sync(0xffffffffu, hit);
    if (!m) continue;
    cnt += __popc(m);
    double2 p = make_double2(0.0, 0.0);
    if (hit) p = obs[i];
    while (m) {                                  // the members in lane order: observation order
      const int b = __ffs(m) - 1;
      m &= m - 1;
      const double vx = __shfl_sync(0xffffffffu, p.x, b), vy = __shfl_sync(0xffffffffu, p.y, b);
      acc = __dadd_rn(acc, lane == 0 ? vx : vy);
    }
  }
  if (lane == 0) { sum->x = acc; *count = cnt; }
  if (lane == 1) sum->y = acc;
}

__global__ void __launch_bounds__(kThreads, 1) kmeans_kernel(const double2* __restrict__ obs, int n, const long long* __restrict__ init_idx,
                                                            int k, int restarts, double thresh, int max_iter, double* __restrict__ books,
                                                            int* __restrict__ book_k, double* __restrict__ dists, int* __restrict__ iters,
                                                            int* __restrict__ best, int* __restrict__ status, unsigned char* __restrict__ ws,
                                                            Layout lay) {
  __shared__ double2 s_book[MYOLO_KMEANS_KMAX], s_sum[MYOLO_KMEANS_KMAX];
  __shared__ int s_cnt[MYOLO_KMEANS_KMAX];
  __shared__ double s_total;
  __shared__ int s_kc, s_go, s_bad;
  __shared__ bool s_last;
  const int r = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  unsigned int* done = reinterpret_cast<unsigned int*>(ws);
  unsigned char* mine = ws + kHeader + r * lay.stride;
  int* starts = reinterpret_cast<int*>(mine + lay.starts_off);
  double* part = reinterpret_cast<double*>(mine + lay.part_off);
  unsigned char* code = mine + lay.codes_off;
  const int n_leaves = (int)lay.leaves;

  if (threadIdx.x == 0) { s_kc = k; s_bad = 0; s_go = CUDART_INF > thresh; }   // scipy's `while diff > thresh` from diff = inf
  __syncthreads();
  if (threadIdx.x < k) {
    const long long j = init_idx[(long long)r * k + threadIdx.x];
    if (j < 0 || j >= n) s_bad = 1;
    else s_book[threadIdx.x] = obs[j];
  }
  if (threadIdx.x == 32) enumerate_leaves(n, starts);
  __syncthreads();
  double prev = CUDART_INF;     // thread 0's
  int it = 0;
  if (!s_bad) {
    for (;;) {
      vq_leaves(obs, starts, n_leaves, s_book, s_kc, code, part);
      __syncthreads();
      const int kc = s_kc;
      if (!s_go) {                                         // the final vq: its mean is the restart's distortion
        if (threadIdx.x == 0) s_total = tree_sum(n, part);
        break;
      }
      if (warp < kc) cluster_sum(obs, code, n, warp, lane, &s_sum[warp], &s_cnt[warp]);
      if (warp == kWarps - 1 && lane == 0) s_total = tree_sum(n, part);   // overlaps the other warps' cluster sums
      __syncthreads();
      if (threadIdx.x == 0) {
        const double cur = __ddiv_rn(s_total, (double)n);
        int kn = 0;
        for (int j = 0; j < kc; ++j)
          if (s_cnt[j] > 0) {
            s_book[kn] = make_double2(__ddiv_rn(s_sum[j].x, (double)s_cnt[j]), __ddiv_rn(s_sum[j].y, (double)s_cnt[j]));
            ++kn;
          }
        s_kc = kn;
        const double diff = fabs(prev - cur);
        prev = cur;
        ++it;
        s_go = diff > thresh;
        if (s_go && it >= max_iter) { s_go = 0; s_bad = 2; }  // the iteration cap: the final vq still runs, the status word reports it
      }
      __syncthreads();
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const int kc = s_kc;
    for (int j = 0; j < k; ++j) {
      const double2 b = j < kc ? s_book[j] : make_double2(0.0, 0.0);
      books[((long long)r * k + j) * 2] = b.x;
      books[((long long)r * k + j) * 2 + 1] = b.y;
    }
    book_k[r] = s_bad == 1 ? 0 : kc;
    dists[r] = s_bad == 1 ? CUDART_NAN : __ddiv_rn(s_total, (double)n);
    iters[r] = it;
    if (s_bad) atomicOr(status, s_bad == 1 ? MYOLO_KMEANS_BAD_INDEX : MYOLO_KMEANS_MAX_ITER);
    __threadfence();
    s_last = atomicAdd(done, 1u) == (unsigned)restarts - 1;
  }
  __syncthreads();
  if (s_last && threadIdx.x == 0) {                        // every restart's result is visible: pick the first strict minimum
    __threadfence();
    double bd = CUDART_INF;
    int bi = -1;
    for (int q = 0; q < restarts; ++q) {
      const double d = __ldcg(dists + q);
      if (d < bd) { bd = d; bi = q; }
    }
    *best = bi;
  }
}

int kmeans_ctas(int* ctas) {
  int dev = 0, sms = 0, per_sm = 0;
  MYOLO_CHECK_CUDA(cudaGetDevice(&dev));
  MYOLO_CHECK_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  MYOLO_CHECK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kmeans_kernel, kThreads, 0));
  MYOLO_REQUIRE(per_sm > 0, "kmeans: the kernel cannot be resident");
  *ctas = per_sm * sms;
  return 0;
}

}  // namespace

}  // namespace myolo

using namespace myolo;

extern "C" int64_t myolo_kmeans_workspace_bytes(int64_t n, int k, int restarts) {
  if (n < 1 || n >= (int64_t(1) << 30) || k < 1 || restarts < 1) return -1;
  return kHeader + (int64_t)restarts * layout(n).stride;
}

extern "C" int myolo_kmeans(const double* obs, int64_t n, int d, const int64_t* init_idx, int k, int restarts, double thresh, int max_iter,
                            double* books, int32_t* book_k, double* dists, int32_t* iters, int32_t* best, int32_t* status, void* ws,
                            int64_t ws_bytes, void* stream) {
  NvtxRange nvtx_("myolo_kmeans");
  MYOLO_REQUIRE(obs && init_idx && books && book_k && dists && iters && best && status && ws && restarts >= 1 && max_iter >= 1,
                "kmeans: bad arguments");
  MYOLO_REQUIRE(d == 2, "kmeans: d = %d features, only d = 2 is built", d);
  MYOLO_REQUIRE(k >= 1 && k <= MYOLO_KMEANS_KMAX, "kmeans: k = %d, needs 1 <= k <= %d", k, MYOLO_KMEANS_KMAX);
  MYOLO_REQUIRE(n >= k && n < (int64_t(1) << 30), "kmeans: n = %lld observations, needs k <= n < 2^30", (long long)n);
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  int ctas = 0;
  int rc = kmeans_ctas(&ctas);
  if (rc) return rc;
  MYOLO_REQUIRE(restarts <= ctas, "kmeans: %d restarts, at most %d (one co-resident CTA each)", restarts, ctas);
  MYOLO_REQUIRE(ws_bytes >= myolo_kmeans_workspace_bytes(n, k, restarts), "kmeans: workspace too small");
  MYOLO_CHECK_CUDA(cudaMemsetAsync(ws, 0, sizeof(unsigned int), s));
  MYOLO_CHECK_CUDA(cudaMemsetAsync(status, 0, sizeof(int32_t), s));
  kmeans_kernel<<<restarts, kThreads, 0, s>>>(reinterpret_cast<const double2*>(obs), (int)n, reinterpret_cast<const long long*>(init_idx),
                                              k, restarts, thresh, max_iter, books, book_k, dists, iters, best, status,
                                              static_cast<unsigned char*>(ws), layout(n));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
