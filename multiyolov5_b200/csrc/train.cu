// Training-mode kernels (see train.h).  Correct-first implementations: the data gradients of all convolutions reuse the wgmma
// implicit-GEMM kernel (a conv of dY with flipped/transposed weights); weight gradients run on legacy mma.sync with split-K
// atomics; everything else is plain coalesced CUDA.  Reference semantics: torch.autograd through models/common.py / models/yolo.py
// in train mode (BatchNorm with batch statistics, eps 1e-3, momentum 0.03: reference utils/torch_utils.py:150-152).
#include <algorithm>
#include <climits>

#include "train.h"

namespace myolo {

static inline int grid_for_t(long items, int block, int max_blocks = 132 * 32) {
  long b = (items + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}
__device__ __forceinline__ __half* tv(const TensorView& v, int b, int y, int x) {
  return reinterpret_cast<__half*>(v.base) + (((size_t)b * v.H + y) * v.W + x) * v.ctot;
}
__device__ __forceinline__ float* tvf(const TensorView& v, int b, int y, int x) {
  return reinterpret_cast<float*>(v.base) + (((size_t)b * v.H + y) * v.W + x) * v.ctot;
}
__device__ __forceinline__ float ldv(const TensorView& v, int b, int y, int x, int c) {
  return v.dtype == MYOLO_F32 ? tvf(v, b, y, x)[c] : __half2float(tv(v, b, y, x)[c]);
}
__device__ __forceinline__ void stv(const TensorView& v, int b, int y, int x, int c, float f) {
  if (v.dtype == MYOLO_F32) tvf(v, b, y, x)[c] = f;
  else tv(v, b, y, x)[c] = __float2half_rn(f);
}
// the per-channel shift of the BN statistics sums: the value at the centre pixel of image 0 (an interior pixel: a corner, the first
// pixel, sees the zero padding of every 3x3 conv before it and on flat content lies farther from the mean than 0 does)
__device__ __forceinline__ const __half* bn_shift_ptr(const TensorView& u) {
  return reinterpret_cast<const __half*>(u.base) + ((size_t)(u.H / 2) * u.W + u.W / 2) * u.ctot;
}
__device__ __forceinline__ float act_fwd(float z, int act) {
  if (act == MYOLO_ACT_SILU) return z / (1.0f + __expf(-z));
  if (act == MYOLO_ACT_SIGMOID) return 1.0f / (1.0f + __expf(-z));
  return z;
}
__device__ __forceinline__ float act_grad(float z, int act) {   // d act(z) / dz
  if (act == MYOLO_ACT_SILU) {
    const float s = 1.0f / (1.0f + __expf(-z));
    return s * (1.0f + z * (1.0f - s));
  }
  if (act == MYOLO_ACT_SIGMOID) {
    const float s = 1.0f / (1.0f + __expf(-z));
    return s * (1.0f - s);
  }
  return 1.0f;
}

// ------------------------------------------------------------------------------------------------
// per-channel reductions over all pixels of an NHWC view:  out[k][c] = sum_p f_k(p, c)
//   grid.x = channel groups of 32, grid.y = pixel slabs; each block reduces its slab and atomically adds 1 or 2 sums per channel
// ------------------------------------------------------------------------------------------------
template <int MODE>   // 0: (sum u, sum u^2)   1: (sum dz, sum dz*xhat) for BN backward   2: (sum dy) column sum (bias gradient)
__global__ void chan_reduce_kernel(TensorView a, TensorView bview, const float* __restrict__ stats, const float* __restrict__ gamma,
                                   const float* __restrict__ beta, int act, float* out, long npix, int C) {
  __shared__ float sh[2][8][32];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int lane_p = threadIdx.x >> 5;                      // 8 pixel lanes
  const long per = (npix + gridDim.y - 1) / gridDim.y;
  const long p0 = (long)blockIdx.y * per, p1 = min(npix, p0 + per);
  float s0 = 0.f, s1 = 0.f;
  if (c < C) {
    float mean = 0.f, istd = 0.f, g = 0.f, bt = 0.f;
    if (MODE == 1) { mean = stats[c]; istd = stats[C + c]; g = gamma[c]; bt = beta[c]; }
    const float shift = MODE == 0 ? __half2float(bn_shift_ptr(a)[c]) : 0.f;     // MODE 0 sums u - shift (see chan_reduce_v_kernel)
    for (long p = p0 + lane_p; p < p1; p += 8) {
      const size_t off = (size_t)p * a.ctot + c;
      if (MODE == 0) {
        const float u = __half2float(reinterpret_cast<const __half*>(a.base)[off]) - shift;
        s0 += u; s1 += u * u;
      } else if (MODE == 1) {
        const float xh = (__half2float(reinterpret_cast<const __half*>(a.base)[off]) - mean) * istd;
        const float dy = __half2float(reinterpret_cast<const __half*>(bview.base)[(size_t)p * bview.ctot + c]);
        const float dz = dy * act_grad(g * xh + bt, act);
        s0 += dz; s1 += dz * xh;
      } else {
        s0 += a.dtype == MYOLO_F32 ? reinterpret_cast<const float*>(a.base)[off] : __half2float(reinterpret_cast<const __half*>(a.base)[off]);
      }
    }
  }
  sh[0][lane_p][threadIdx.x & 31] = s0;
  sh[1][lane_p][threadIdx.x & 31] = s1;
  __syncthreads();
  if (lane_p == 0 && c < C) {
    for (int l = 1; l < 8; ++l) { s0 += sh[0][l][threadIdx.x & 31]; s1 += sh[1][l][threadIdx.x & 31]; }
    atomicAdd(out + c, s0);
    if (MODE != 2) atomicAdd(out + C + c, s1);
  }
}

// Vectorised variant for fp16 views (the BN forward statistics and the BN backward sums): a thread owns 8 channels (one 16-byte load
// per pixel), the block's threads tile (pixel lanes x channel vectors) so a pixel's channels are read as one contiguous run; per-block
// partials are combined through shared memory and added atomically; the LAST block to finish (ticket) runs the per-channel epilogue:
//   MODE 0: mean / inverse std -> stats, running-statistics update        MODE 1: dgamma += sum(dz*xhat), dbeta += sum(dz)
// MODE 0 sums d = u - shift and d^2 with shift = one of the channel's own values (bn_shift_ptr): var = E[d^2] - E[d]^2 then cancels only
// on the distance of the mean from that value.  Summing u itself loses the variance of a channel whose mean is large against its spread
// (flat image content: letterbox padding, sky, road): at mean/std = 200 the fp32 E[u^2] - mean^2 is off by ~1e-2 of the normalised output.
// final_out (MODE 0, deferred running statistics): batch mean and biased variance; (MODE 1): the two sums.
// rec (MODE 0, synchronised BN): the epilogue writes this rank's record {count, mean[C], biased var[C]} (bn_sync_combine_kernel) and
// finalises nothing.
// mean / inverse std and the running-statistics update of one channel from the batch mean and biased variance of n values: shared by the
// local epilogue and the synchronised combine, so that a combine over one record repeats the local path bit for bit
__device__ __forceinline__ void bn_finalize_channel(float mean, float var, float n, const BnParams& bn, int c, int C, float* stats_out) {
  stats_out[c] = mean;
  stats_out[C + c] = rsqrtf(var + bn.eps);
  if (bn.running_mean) {                                       // running stats: unbiased variance, momentum 0.03
    bn.running_mean[c] = (1.f - bn.momentum) * bn.running_mean[c] + bn.momentum * mean;
    bn.running_var[c] = (1.f - bn.momentum) * bn.running_var[c] + bn.momentum * var * (n / fmaxf(n - 1.f, 1.f));
  }
}
template <int MODE>
__global__ void __launch_bounds__(256) chan_reduce_v_kernel(TensorView a, TensorView bview, const float* __restrict__ stats,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                                            float* out, long npix, int C, BnParams bn, float* stats_out,
                                                            unsigned* ticket, float* final_out, float* rec) {
  __shared__ float sh[2][2048];
  __shared__ int is_last;
  pdl_enter();
  const int nv = C >> 3, lanes = 256 / nv;
  const int t = threadIdx.x;
  const bool active = t < lanes * nv;
  const int cv = active ? t % nv : 0, lane = active ? t / nv : 0;
  float s0[8], s1[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) { s0[k] = 0.f; s1[k] = 0.f; }
  if (active) {
    float mean[8], istd[8], g[8], bt[8];
    if (MODE == 1) {
#pragma unroll
      for (int k = 0; k < 8; ++k) { const int c = cv * 8 + k; mean[k] = stats[c]; istd[k] = stats[C + c]; g[k] = gamma[c]; bt[k] = beta[c]; }
    }
    const __half* ab = reinterpret_cast<const __half*>(a.base);
    const __half* bb = reinterpret_cast<const __half*>(bview.base);
    float shift[8];
    if (MODE == 0) {
      const uint4 q0 = *reinterpret_cast<const uint4*>(bn_shift_ptr(a) + cv * 8);
#pragma unroll
      for (int k = 0; k < 8; ++k) shift[k] = __half2float(reinterpret_cast<const __half*>(&q0)[k]);
    }
    for (long p = (long)blockIdx.x * lanes + lane; p < npix; p += (long)gridDim.x * lanes) {
      const uint4 q = *reinterpret_cast<const uint4*>(ab + (size_t)p * a.ctot + cv * 8);
      const __half* h = reinterpret_cast<const __half*>(&q);
      if (MODE == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { const float u = __half2float(h[k]) - shift[k]; s0[k] += u; s1[k] += u * u; }
      } else {
        const uint4 r = *reinterpret_cast<const uint4*>(bb + (size_t)p * bview.ctot + cv * 8);
        const __half* hr = reinterpret_cast<const __half*>(&r);
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          const float xh = (__half2float(h[k]) - mean[k]) * istd[k];
          const float dz = __half2float(hr[k]) * act_grad(g[k] * xh + bt[k], act);
          s0[k] += dz; s1[k] += dz * xh;
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) { sh[0][lane * C + cv * 8 + k] = s0[k]; sh[1][lane * C + cv * 8 + k] = s1[k]; }
  }
  __syncthreads();
  for (int c = t; c < C; c += 256) {
    float x0 = 0.f, x1 = 0.f;
    for (int l = 0; l < lanes; ++l) { x0 += sh[0][l * C + c]; x1 += sh[1][l * C + c]; }
    atomicAdd(out + c, x0);
    atomicAdd(out + C + c, x1);
  }
  __threadfence();
  __syncthreads();
  if (t == 0) is_last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // the last block consumes the sums and leaves accumulators + ticket ZERO for the next launch on this scratch (allocated zeroed): no
  // memset node between the producing conv and this kernel, so the programmatic-launch edge survives
  if (t == 0) *ticket = 0u;
  if (MODE == 0 && rec && t == 0) reinterpret_cast<int*>(rec)[0] = (int)npix;
  for (int c = t; c < C; c += 256) {
    const float x0 = __ldcg(out + c), x1 = __ldcg(out + C + c);
    out[c] = 0.f;
    out[C + c] = 0.f;
    if (MODE == 0) {
      const float n = (float)npix;
      const float d = x0 / n;
      const float mean = __half2float(bn_shift_ptr(a)[c]) + d;
      const float var = fmaxf(x1 / n - d * d, 0.f);                // biased variance normalises (F.batch_norm, training=True)
      if (rec) { rec[kBnRecHead + c] = mean; rec[kBnRecHead + C + c] = var; continue; }
      if (final_out) { final_out[c] = mean; final_out[C + c] = var; }
      bn_finalize_channel(mean, var, n, bn, c, C, stats_out);
    } else {
      if (final_out) { final_out[c] = x0; final_out[C + c] = x1; }
      // parameter gradients are accumulated atomically everywhere: the det and the seg backward of one training step may run concurrently
      if (bn.d_beta) atomicAdd(bn.d_beta + c, x0);
      if (bn.d_gamma) atomicAdd(bn.d_gamma + c, x1);
    }
  }
}
static inline int reduce_v_grid(long npix, int C) {
  const int lanes = 256 / (C / 8);
  return (int)std::max<long>(1, std::min<long>(132 * 2, npix / ((long)lanes * 4)));
}

// sums of u - shift (chan_reduce_kernel<0>): the shift is read back from u
__global__ void bn_finalize_kernel(TensorView u, float* sums, float* stats, BnParams bn, long npix) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= bn.C) return;
  const float n = (float)npix;
  const float d = sums[c] / n;
  const float mean = __half2float(bn_shift_ptr(u)[c]) + d;
  const float var = fmaxf(sums[bn.C + c] / n - d * d, 0.f);                 // biased variance normalises (F.batch_norm, training=True)
  stats[c] = mean;
  stats[bn.C + c] = rsqrtf(var + bn.eps);
  if (bn.running_mean) {                                                       // running stats: unbiased variance, momentum 0.03
    bn.running_mean[c] = (1.f - bn.momentum) * bn.running_mean[c] + bn.momentum * mean;
    bn.running_var[c] = (1.f - bn.momentum) * bn.running_var[c] + bn.momentum * var * (n / fmaxf(n - 1.f, 1.f));
  }
}

// deferred running statistics: one launch applies r <- (1-m) r + m * stat for every BN layer of a plan from the batch mean and biased
// variance its last forward left (computed from shifted sums by chan_reduce_v_kernel<0>)
__global__ void __launch_bounds__(256) bn_apply_running_kernel(const RunningJob* __restrict__ jobs) {
  const RunningJob j = jobs[blockIdx.x];
  const float n = (float)j.npix;
  for (int c = threadIdx.x; c < j.C; c += 256) {
    const float mean = j.batch_stats[c];
    const float var = j.batch_stats[j.C + c];
    j.running_mean[c] = (1.f - j.momentum) * j.running_mean[c] + j.momentum * mean;
    j.running_var[c] = (1.f - j.momentum) * j.running_var[c] + j.momentum * var * (n / fmaxf(n - 1.f, 1.f));
  }
}
int launch_bn_apply_running(const RunningJob* d_jobs, int n_jobs, cudaStream_t s) {
  if (n_jobs <= 0) return 0;
  bn_apply_running_kernel<<<n_jobs, 256, 0, s>>>(d_jobs);
  MYOLO_LAUNCH_CHECK();
  g_launch_count++;
  return 0;
}

int launch_bn_stats(const TensorView& u, const BnParams& bn_in, float* stats, float* scratch, cudaStream_t s, bool defer_running) {
  BnParams bn = bn_in;
  MYOLO_REQUIRE(u.dtype == MYOLO_F16 && bn.set && bn.C == u.C, "bn_stats: bad view / BN parameters not set");
  MYOLO_REQUIRE(!defer_running || (u.C % 8 == 0 && u.C <= 2048 && u.ctot % 8 == 0), "bn_stats: deferred running statistics need C %% 8 == 0");
  if (defer_running) bn.running_mean = bn.running_var = nullptr;     // the sums stay in scratch + 2C for myolo_plan_apply_running
  const long npix = (long)u.B * u.H * u.W;
  // scratch (zero on entry, left zero by the kernel): 2*C sums, 2*C final values (batch mean / variance of a deferring plan, the backward's
  // sums), the completion ticket
  if (u.C % 8 == 0 && u.C <= 2048 && u.ctot % 8 == 0) {
    MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<0>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, u, (const float*)nullptr,
                                (const float*)nullptr, (const float*)nullptr, 0, scratch, npix, u.C, bn, stats,
                                reinterpret_cast<unsigned*>(scratch + 4 * u.C), defer_running ? scratch + 2 * u.C : (float*)nullptr,
                                (float*)nullptr));
    g_launch_count++;
    return 0;
  }
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));
  dim3 g(ceil_div(u.C, 32), (unsigned)std::min<long>(256, std::max<long>(1, npix / 256)));
  chan_reduce_kernel<0><<<g, 256, 0, s>>>(u, u, nullptr, nullptr, nullptr, 0, scratch, npix, u.C);
  MYOLO_LAUNCH_CHECK();
  bn_finalize_kernel<<<ceil_div(u.C, 128), 128, 0, s>>>(u, scratch, stats, bn, npix);
  MYOLO_LAUNCH_CHECK();
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));    // contract of the scratch: zero between launches
  return 0;
}

// ---- synchronised BatchNorm (torch.nn.SyncBatchNorm, torch/nn/modules/_functions.py) ----
static bool bn_sync_shape_ok(const TensorView& u) { return u.dtype == MYOLO_F16 && u.C % 8 == 0 && u.C <= 2048 && u.ctot % 8 == 0; }

int launch_bn_stats_record(const TensorView& u, const BnParams& bn, float* rec, float* scratch, cudaStream_t s) {
  MYOLO_REQUIRE(bn.set && bn.C == u.C && bn_sync_shape_ok(u), "bn_stats_record: synchronised BatchNorm needs an fp16 view with C %% 8 == 0 "
                "and C <= 2048 (C = %d)", u.C);
  const long npix = (long)u.B * u.H * u.W;
  MYOLO_REQUIRE(npix > 0 && npix < (1L << 31), "bn_stats_record: %ld values per channel do not fit the record's int32 count", npix);
  MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<0>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, u, (const float*)nullptr,
                              (const float*)nullptr, (const float*)nullptr, 0, scratch, npix, u.C, bn, (float*)nullptr,
                              reinterpret_cast<unsigned*>(scratch + 4 * u.C), (float*)nullptr, rec));
  g_launch_count++;
  return 0;
}

// Global statistics from the gathered records, combined in rank order with the pairwise (Chan et al.) update in fp64:
//   n = na + nb,  mean = ma + (mb - ma) nb / n,  M2 = M2a + M2b + (mb - ma)^2 na nb / n,  var = M2 / n   (biased)
// One record is passed through unchanged, so the result is the local epilogue's to the bit.  Every rank combines the same records in the
// same order and writes the same bits: running statistics stay identical across ranks.  inv_n = 1 / N for the backward.
__global__ void bn_sync_combine_kernel(const float* __restrict__ recs, int n_rec, int C, BnParams bn, float* stats, float* inv_n) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const long stride = kBnRecHead + 2L * C;
  long n = reinterpret_cast<const int*>(recs)[0];
  float mean = recs[kBnRecHead + c], var = recs[kBnRecHead + C + c];
  if (n_rec > 1) {
    double na = (double)n, ma = mean, m2 = (double)var * na;
    for (int r = 1; r < n_rec; ++r) {
      const float* rr = recs + r * stride;
      const double nb = (double)reinterpret_cast<const int*>(rr)[0];
      const double mb = rr[kBnRecHead + c], m2b = (double)rr[kBnRecHead + C + c] * nb;
      const double nab = na + nb, delta = mb - ma;
      ma += delta * nb / nab;
      m2 += m2b + delta * delta * na * nb / nab;
      na = nab;
    }
    n = (long)na;
    mean = (float)ma;
    var = (float)(m2 / na);
  }
  if (c == 0) *inv_n = 1.0f / (float)n;
  bn_finalize_channel(mean, var, (float)n, bn, c, C, stats);
}
int launch_bn_sync_combine(const float* recs, int n_rec, const BnParams& bn, float* stats, float* inv_n, cudaStream_t s) {
  MYOLO_REQUIRE(recs && n_rec >= 1 && stats && inv_n, "bn_sync_combine: bad arguments");
  bn_sync_combine_kernel<<<ceil_div(bn.C, 128), 128, 0, s>>>(recs, n_rec, bn.C, bn, stats, inv_n);
  MYOLO_LAUNCH_CHECK();
  g_launch_count++;
  return 0;
}

// sums[j] += sums[g * n + j] for g = 1 .. n_groups-1, in group order (the all-reduce of the backward sums between emulated ranks)
__global__ void bn_sync_sum_kernel(float* sums, int n_groups, int n) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  float acc = sums[j];
  for (int g = 1; g < n_groups; ++g) acc += sums[(long)g * n + j];
  sums[j] = acc;
}
int launch_bn_sync_sum(float* sums, int n_groups, int n, cudaStream_t s) {
  if (n_groups <= 1) return 0;
  bn_sync_sum_kernel<<<ceil_div(n, 256), 256, 0, s>>>(sums, n_groups, n);
  MYOLO_LAUNCH_CHECK();
  g_launch_count++;
  return 0;
}

__global__ void bn_act_fwd_kernel(TensorView u, TensorView res, bool has_res, TensorView y, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, const float* __restrict__ stats, int act) {
  pdl_enter();
  const long total = (long)u.B * u.H * u.W * (u.C / 8);
  const int nv = u.C / 8, C = u.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    const long p = i / nv;
    const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(u.base) + (size_t)p * u.ctot + v * 8);
    const __half* h = reinterpret_cast<const __half*>(&q);
    uint4 r = make_uint4(0, 0, 0, 0);
    if (has_res) r = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(res.base) + (size_t)p * res.ctot + v * 8);
    const __half* hr = reinterpret_cast<const __half*>(&r);
    uint4 o;
    __half* ho = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = v * 8 + k;
      const float z = gamma[c] * (__half2float(h[k]) - stats[c]) * stats[C + c] + beta[c];
      float val = act_fwd(z, act);
      if (has_res) val += __half2float(hr[k]);
      ho[k] = __float2half_rn(val);
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(y.base) + (size_t)p * y.ctot + v * 8) = o;
  }
}
int launch_bn_act_fwd(const TensorView& u, const TensorView* res, const TensorView& y, const BnParams& bn, const float* stats, int act,
                      cudaStream_t s) {
  MYOLO_REQUIRE(u.C % 8 == 0 && u.C == y.C && u.ctot % 8 == 0 && y.ctot % 8 == 0 && (!res || (res->C == u.C && res->ctot % 8 == 0)),
                "bn_act_fwd: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(bn_act_fwd_kernel, dim3(grid_for_t((long)u.B * u.H * u.W * (u.C / 8), 256)), dim3(256), 0, s, u, res ? *res : u,
                              res != nullptr, y, (const float*)bn.gamma, (const float*)bn.beta, stats, act));
  g_launch_count++;
  return 0;
}

__global__ void bn_act_bwd_kernel(TensorView u, TensorView dy, TensorView du, TensorView dres, bool has_res, const float* __restrict__ gamma,
                                  const float* __restrict__ beta, const float* __restrict__ stats, const float* __restrict__ sums, int act,
                                  float inv_n_host, const float* __restrict__ inv_n_dev) {
  pdl_enter();
  const float inv_n = inv_n_dev ? *inv_n_dev : inv_n_host;       // synchronised BN: 1 / N over all ranks, from bn_sync_combine_kernel
  const long total = (long)u.B * u.H * u.W * (u.C / 8);
  const int nv = u.C / 8, C = u.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    const long p = i / nv;
    const uint4 q = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(u.base) + (size_t)p * u.ctot + v * 8);
    const uint4 g = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(dy.base) + (size_t)p * dy.ctot + v * 8);
    const __half* h = reinterpret_cast<const __half*>(&q);
    const __half* hg = reinterpret_cast<const __half*>(&g);
    uint4 o;
    __half* ho = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = v * 8 + k;
      const float xh = (__half2float(h[k]) - stats[c]) * stats[C + c];
      const float dz = __half2float(hg[k]) * act_grad(gamma[c] * xh + beta[c], act);
      ho[k] = __float2half_rn(gamma[c] * stats[C + c] * (dz - sums[c] * inv_n - xh * sums[C + c] * inv_n));
    }
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(du.base) + (size_t)p * du.ctot + v * 8) = o;
    if (has_res) {                                              // shortcut gradient: d(residual) += dy
      uint4* dp = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(dres.base) + (size_t)p * dres.ctot + v * 8);
      uint4 r = *dp;
      __half2* hr = reinterpret_cast<__half2*>(&r);
      const __half2* hb = reinterpret_cast<const __half2*>(&g);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 fa = __half22float2(hr[k]), fb = __half22float2(hb[k]);
        hr[k] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
      }
      *dp = r;
    }
  }
}
__global__ void bn_param_grad_kernel(const float* sums, BnParams bn) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= bn.C) return;
  if (bn.d_beta) atomicAdd(bn.d_beta + c, sums[c]);
  if (bn.d_gamma) atomicAdd(bn.d_gamma + c, sums[bn.C + c]);
}
__global__ void add_acc_kernel(TensorView dst, TensorView src) {   // dst += src (fp16 NHWC)
  const long total = (long)dst.B * dst.H * dst.W * (dst.C / 8);
  const int nv = dst.C / 8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    const long p = i / nv;
    uint4* dp = reinterpret_cast<uint4*>(reinterpret_cast<__half*>(dst.base) + (size_t)p * dst.ctot + v * 8);
    uint4 a = *dp;
    const uint4 b = *reinterpret_cast<const uint4*>(reinterpret_cast<const __half*>(src.base) + (size_t)p * src.ctot + v * 8);
    __half2* ha = reinterpret_cast<__half2*>(&a);
    const __half2* hb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 fa = __half22float2(ha[k]), fb = __half22float2(hb[k]);
      ha[k] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
    }
    *dp = a;
  }
}
int launch_bn_bwd_sums(const TensorView& u, const TensorView& dy, const BnParams& bn, const float* stats, int act, float* scratch,
                       float* sums_out, cudaStream_t s) {
  MYOLO_REQUIRE(bn_sync_shape_ok(u) && dy.C == u.C && dy.ctot % 8 == 0, "bn_bwd_sums: synchronised BatchNorm needs C %% 8 == 0 and C <= 2048");
  const long npix = (long)u.B * u.H * u.W;
  MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<1>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, dy, stats, (const float*)bn.gamma,
                              (const float*)bn.beta, act, scratch, npix, u.C, bn, (float*)nullptr,
                              reinterpret_cast<unsigned*>(scratch + 4 * u.C), sums_out, (float*)nullptr));
  g_launch_count++;
  return 0;
}

int launch_bn_act_bwd(const TensorView& u, const TensorView& dy, const TensorView& du, const TensorView* d_res, const BnParams& bn,
                      const float* stats, int act, float* scratch, cudaStream_t s, const float* synced_sums, const float* inv_n) {
  MYOLO_REQUIRE(u.C % 8 == 0 && dy.C == u.C && du.C == u.C && dy.ctot % 8 == 0 && du.ctot % 8 == 0 && u.ctot % 8 == 0, "bn_act_bwd: bad views");
  MYOLO_REQUIRE(!d_res || (d_res->C == u.C && d_res->ctot % 8 == 0), "bn_act_bwd: bad residual gradient view");
  MYOLO_REQUIRE(!synced_sums == !inv_n, "bn_act_bwd: synchronised sums and 1 / N go together");
  const long npix = (long)u.B * u.H * u.W;
  const float* sums = scratch;
  if (synced_sums) {
    sums = synced_sums;                  // launch_bn_bwd_sums + the exchange already ran
  } else if (u.C <= 2048) {
    MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<1>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, dy, stats, (const float*)bn.gamma,
                                (const float*)bn.beta, act, scratch, npix, u.C, bn, (float*)nullptr,
                                reinterpret_cast<unsigned*>(scratch + 4 * u.C), scratch + 2 * u.C, (float*)nullptr));
    g_launch_count++;
    sums = scratch + 2 * u.C;            // the reduce kernel leaves its accumulators zero and hands the totals over here
  } else {
    MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));
    dim3 g(ceil_div(u.C, 32), (unsigned)std::min<long>(256, std::max<long>(1, npix / 256)));
    chan_reduce_kernel<1><<<g, 256, 0, s>>>(u, dy, stats, bn.gamma, bn.beta, act, scratch, npix, u.C);
    MYOLO_LAUNCH_CHECK();
    bn_param_grad_kernel<<<ceil_div(u.C, 128), 128, 0, s>>>(scratch, bn);
    MYOLO_LAUNCH_CHECK();
  }
  MYOLO_CHECK_CUDA(launch_pdl(bn_act_bwd_kernel, dim3(grid_for_t(npix * (u.C / 8), 256)), dim3(256), 0, s, u, dy, du, d_res ? *d_res : du,
                              d_res != nullptr, (const float*)bn.gamma, (const float*)bn.beta, stats, sums, act, 1.0f / (float)npix, inv_n));
  g_launch_count++;
  if (sums == scratch) MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));   // (> 2048 channels: generic path)
  return 0;
}

// dst += src (any dtype through ldv/stv; used by the ADD backward)
__global__ void grad_add_kernel(TensorView src, TensorView dst) {
  const long total = (long)dst.B * dst.H * dst.W * dst.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dst.C);
    long q = i / dst.C;
    const int x = (int)(q % dst.W); q /= dst.W;
    const int y = (int)(q % dst.H);
    const int b = (int)(q / dst.H);
    stv(dst, b, y, x, c, ldv(dst, b, y, x, c) + ldv(src, b, y, x, c));
  }
}
int launch_grad_add(const TensorView& src, const TensorView& dst, cudaStream_t s) {
  MYOLO_REQUIRE(src.C == dst.C && src.H == dst.H && src.W == dst.W, "grad_add: shape mismatch");
  grad_add_kernel<<<grid_for_t((long)dst.B * dst.H * dst.W * dst.C, 256), 256, 0, s>>>(src, dst);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
// din[b,0,0,c] += sum_{y,x} dout[b,y,x,c]   (one block per (image, 32 channels))
__global__ void broadcast_bwd_kernel(TensorView dout, TensorView din) {
  __shared__ float sh[8][32];
  const int ncg = (dout.C + 31) / 32;
  const int cg = blockIdx.x % ncg, b = blockIdx.x / ncg;
  const int c = cg * 32 + (threadIdx.x & 31), lp = threadIdx.x >> 5;
  float acc = 0.f;
  if (c < dout.C)
    for (int p = lp; p < dout.H * dout.W; p += 8) acc += ldv(dout, b, p / dout.W, p % dout.W, c);
  sh[lp][threadIdx.x & 31] = acc;
  __syncthreads();
  if (lp == 0 && c < dout.C) {
    for (int l = 1; l < 8; ++l) acc += sh[l][threadIdx.x & 31];
    stv(din, b, 0, 0, c, ldv(din, b, 0, 0, c) + acc);
  }
}
int launch_broadcast_bwd(const TensorView& dout, const TensorView& din, cudaStream_t s) {
  MYOLO_REQUIRE(din.H == 1 && din.W == 1 && din.C == dout.C, "broadcast_bwd: bad views");
  broadcast_bwd_kernel<<<dout.B * ceil_div(dout.C, 32), 256, 0, s>>>(dout, din);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// dropout (train mode): keep mask from a counter-based hash - the backward pass regenerates it instead of storing it.
// (PyTorch's Philox stream cannot be reproduced bit for bit; the mask is Bernoulli(1-p) per element, like nn.Dropout.)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ bool dropout_keep(unsigned long long seed, unsigned long long step, unsigned salt, unsigned long long idx, float p) {
  unsigned long long z = seed ^ (step * 0x9E3779B97F4A7C15ull) ^ ((unsigned long long)salt << 48) ^ (idx * 0xD1B54A32D192ED03ull);
  z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull;          // splitmix64 finaliser
  z ^= z >> 27; z *= 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f) >= p;
}
__global__ void dropout_kernel(TensorView x, TensorView y, float p, unsigned long long seed, const unsigned long long* step, unsigned salt,
                               int accumulate) {
  const long total = (long)x.B * x.H * x.W * x.C;
  const unsigned long long st = *step;
  const float scale = 1.0f / (1.0f - p);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % x.C);
    long q = i / x.C;
    const int xx = (int)(q % x.W); q /= x.W;
    const int yy = (int)(q % x.H);
    const int b = (int)(q / x.H);
    const float v = dropout_keep(seed, st, salt, (unsigned long long)i, p) ? ldv(x, b, yy, xx, c) * scale : 0.f;
    stv(y, b, yy, xx, c, accumulate ? ldv(y, b, yy, xx, c) + v : v);
  }
}
// forward: y = dropout(x);  backward (accumulate = 1): dx += dropout-mask(dy)  (same seed / step / salt -> same mask)
int launch_dropout(const TensorView& x, const TensorView& y, float p, unsigned long long seed, const unsigned long long* step, unsigned salt,
                   int accumulate, cudaStream_t s) {
  MYOLO_REQUIRE(x.C == y.C && x.H == y.H && x.W == y.W && p >= 0.f && p < 1.f && step, "dropout: bad arguments");
  dropout_kernel<<<grid_for_t((long)x.B * x.H * x.W * x.C, 256), 256, 0, s>>>(x, y, p, seed, step, salt, accumulate);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
__global__ void bump_step_kernel(unsigned long long* step) { *step += 1; }
int launch_bump_step(unsigned long long* step, cudaStream_t s) {
  bump_step_kernel<<<1, 1, 0, s>>>(step);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// small elementwise ops (generic dtype through ldv/stv: used on tiny maps or fp32 head buffers)
// ------------------------------------------------------------------------------------------------
__global__ void act_fwd_kernel(TensorView x, TensorView y, int act) {
  const long total = (long)x.B * x.H * x.W * x.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % x.C);
    long p = i / x.C;
    const int xx = (int)(p % x.W); p /= x.W;
    const int yy = (int)(p % x.H);
    const int b = (int)(p / x.H);
    stv(y, b, yy, xx, c, act_fwd(ldv(x, b, yy, xx, c), act));
  }
}
int launch_act_fwd(const TensorView& x, const TensorView& y, int act, cudaStream_t s) {
  act_fwd_kernel<<<grid_for_t((long)x.B * x.H * x.W * x.C, 256), 256, 0, s>>>(x, y, act);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
__global__ void act_bwd_kernel(TensorView x, TensorView dy, TensorView dx, int act) {
  const long total = (long)x.B * x.H * x.W * x.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % x.C);
    long p = i / x.C;
    const int xx = (int)(p % x.W); p /= x.W;
    const int yy = (int)(p % x.H);
    const int b = (int)(p / x.H);
    stv(dx, b, yy, xx, c, ldv(dx, b, yy, xx, c) + ldv(dy, b, yy, xx, c) * act_grad(ldv(x, b, yy, xx, c), act));
  }
}
int launch_act_bwd(const TensorView& x, const TensorView& dy, const TensorView& dx, int act, cudaStream_t s) {
  act_bwd_kernel<<<grid_for_t((long)x.B * x.H * x.W * x.C, 256), 256, 0, s>>>(x, dy, dx, act);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void channel_scale_oop_kernel(TensorView f, TensorView a, TensorView out) {
  const long total = (long)f.B * f.H * f.W * f.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % f.C);
    long p = i / f.C;
    const int x = (int)(p % f.W); p /= f.W;
    const int y = (int)(p % f.H);
    const int b = (int)(p / f.H);
    const float fv = ldv(f, b, y, x, c);
    stv(out, b, y, x, c, fmaf(fv, ldv(a, b, 0, 0, c), fv));
  }
}
int launch_channel_scale_oop(const TensorView& f, const TensorView& a, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(a.H == 1 && a.W == 1 && a.C >= f.C && out.C == f.C, "channel_scale_oop: bad views");
  channel_scale_oop_kernel<<<grid_for_t((long)f.B * f.H * f.W * f.C, 256), 256, 0, s>>>(f, a, out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
// df += dout*(1+a);  da[b,c] += sum_p dout*f    (block = (b, 32-channel group, pixel slab); da is accumulated atomically when fp32)
__global__ void channel_scale_bwd_kernel(TensorView f, TensorView a, TensorView dout, TensorView df, TensorView da) {
  __shared__ float sh[8][32];
  const int ncg = (f.C + 31) / 32;
  const int cg = blockIdx.x % ncg, b = blockIdx.x / ncg;
  const int c = cg * 32 + (threadIdx.x & 31), lp = threadIdx.x >> 5;
  const int npix = f.H * f.W;
  const int per = (npix + gridDim.y - 1) / gridDim.y;
  const int p0 = blockIdx.y * per, p1 = min(npix, p0 + per);
  float acc = 0.f;
  if (c < f.C) {
    const float sc = 1.0f + ldv(a, b, 0, 0, c);
    for (int p = p0 + lp; p < p1; p += 8) {
      const int y = p / f.W, x = p % f.W;
      const float g = ldv(dout, b, y, x, c);
      acc += g * ldv(f, b, y, x, c);
      stv(df, b, y, x, c, ldv(df, b, y, x, c) + g * sc);
    }
  }
  sh[lp][threadIdx.x & 31] = acc;
  __syncthreads();
  if (lp == 0 && c < f.C) {
    for (int l = 1; l < 8; ++l) acc += sh[l][threadIdx.x & 31];
    if (da.dtype == MYOLO_F32) atomicAdd(reinterpret_cast<float*>(da.base) + (size_t)b * da.H * da.W * da.ctot + c, acc);
    else stv(da, b, 0, 0, c, ldv(da, b, 0, 0, c) + acc);
  }
}
int launch_channel_scale_bwd(const TensorView& f, const TensorView& a, const TensorView& dout, const TensorView& df, const TensorView& da,
                             cudaStream_t s) {
  MYOLO_REQUIRE(da.H == 1 && da.W == 1 && a.H == 1 && a.W == 1, "channel_scale_bwd: attention must be a 1x1 map");
  const int slabs = da.dtype == MYOLO_F32 ? std::max(1, std::min(64, f.H * f.W / 64)) : 1;
  channel_scale_bwd_kernel<<<dim3(f.B * ceil_div(f.C, 32), slabs), 256, 0, s>>>(f, a, dout, df, da);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void nearest2x_bwd_kernel(TensorView dout, TensorView din) {
  const long total = (long)din.B * din.H * din.W * din.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % din.C);
    long p = i / din.C;
    const int x = (int)(p % din.W); p /= din.W;
    const int y = (int)(p % din.H);
    const int b = (int)(p / din.H);
    const float g = ldv(dout, b, 2 * y, 2 * x, c) + ldv(dout, b, 2 * y, 2 * x + 1, c) + ldv(dout, b, 2 * y + 1, 2 * x, c) +
                    ldv(dout, b, 2 * y + 1, 2 * x + 1, c);
    stv(din, b, y, x, c, ldv(din, b, y, x, c) + g);
  }
}
int launch_nearest2x_bwd(const TensorView& dout, const TensorView& din, cudaStream_t s) {
  MYOLO_REQUIRE(dout.H == 2 * din.H && dout.W == 2 * din.W && dout.C == din.C, "nearest2x_bwd: bad views");
  nearest2x_bwd_kernel<<<grid_for_t((long)din.B * din.H * din.W * din.C, 256), 256, 0, s>>>(dout, din);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// adjoint of bilinear(align_corners=True): every source pixel gathers from the destination pixels that read it
__device__ __forceinline__ void lerp_src(int dst, int n_in, int n_out, int* i0, int* i1, float* l0, float* l1) {
  const float scale = n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.f;
  const float src = scale * (float)dst;
  *i0 = min((int)src, n_in - 1);
  *i1 = *i0 + (*i0 < n_in - 1 ? 1 : 0);
  *l1 = src - (float)*i0;
  *l0 = 1.0f - *l1;
}
__device__ __forceinline__ void dst_range(int src_i, int n_in, int n_out, int* lo, int* hi) {
  // destination indices d whose i0 or i1 can equal src_i: src(d) in (src_i-1, src_i+1)
  if (n_out <= 1 || n_in <= 1) { *lo = 0; *hi = n_out - 1; return; }
  const float inv = (float)(n_out - 1) / (float)(n_in - 1);
  *lo = max(0, (int)floorf((src_i - 1) * inv) - 1);
  *hi = min(n_out - 1, (int)ceilf((src_i + 1) * inv) + 1);
}
// separable adjoint: tmp[b,sy,dx,c] = sum_dy wy(dy->sy) dout[b,dy,dx,c]  (fp32 scratch), then din[b,sy,sx,c] += sum_dx wx(dx->sx) tmp
__global__ void bilinear_bwd_rows_kernel(TensorView dout, int in_h, float* __restrict__ tmp) {
  const long total = (long)dout.B * in_h * dout.W * dout.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dout.C);
    long p = i / dout.C;
    const int dx = (int)(p % dout.W); p /= dout.W;
    const int sy = (int)(p % in_h);
    const int b = (int)(p / in_h);
    int lo, hi;
    dst_range(sy, in_h, dout.H, &lo, &hi);
    float acc = 0.f;
    for (int dy = lo; dy <= hi; ++dy) {
      int a0, a1; float w0, w1;
      lerp_src(dy, in_h, dout.H, &a0, &a1, &w0, &w1);
      const float wy = (a0 == sy ? w0 : 0.f) + (a1 == sy ? w1 : 0.f);
      if (wy != 0.f) acc += wy * ldv(dout, b, dy, dx, c);
    }
    tmp[i] = acc;
  }
}
__global__ void bilinear_bwd_cols_kernel(const float* __restrict__ tmp, int out_w, TensorView din) {
  const long total = (long)din.B * din.H * din.W * din.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % din.C);
    long p = i / din.C;
    const int sx = (int)(p % din.W); p /= din.W;
    const int sy = (int)(p % din.H);
    const int b = (int)(p / din.H);
    int lo, hi;
    dst_range(sx, din.W, out_w, &lo, &hi);
    float acc = 0.f;
    const float* row = tmp + (((size_t)b * din.H + sy) * out_w) * din.C + c;
    for (int dx = lo; dx <= hi; ++dx) {
      int b0, b1; float v0, v1;
      lerp_src(dx, din.W, out_w, &b0, &b1, &v0, &v1);
      const float wx = (b0 == sx ? v0 : 0.f) + (b1 == sx ? v1 : 0.f);
      if (wx != 0.f) acc += wx * row[(size_t)dx * din.C];
    }
    stv(din, b, sy, sx, c, ldv(din, b, sy, sx, c) + acc);
  }
}
size_t bilinear_bwd_scratch_bytes(const TensorView& dout, const TensorView& din) {
  return (size_t)dout.B * din.H * dout.W * dout.C * sizeof(float);
}
int launch_bilinear_bwd(const TensorView& dout, const TensorView& din, float* scratch, cudaStream_t s) {
  MYOLO_REQUIRE(dout.C == din.C && scratch, "bilinear_bwd: bad views");
  bilinear_bwd_rows_kernel<<<grid_for_t((long)dout.B * din.H * dout.W * dout.C, 256), 256, 0, s>>>(dout, din.H, scratch);
  MYOLO_LAUNCH_CHECK();
  bilinear_bwd_cols_kernel<<<grid_for_t((long)din.B * din.H * din.W * din.C, 128), 128, 0, s>>>(scratch, dout.W, din);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// SPP: the three pools are max pools of the SAME input x with windows 5/9/13 (cascade == direct); each output routes its gradient
// to the first maximum of its window in row-major scan order (ATen max_pool2d backward).  fp32 scratch accumulates, then dx += scratch.
__global__ void spp_bwd_scatter_kernel(TensorView x, TensorView dout3, float* scratch) {
  const long total = (long)x.B * x.H * x.W * x.C * 3;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % x.C);
    long p = i / x.C;
    const int k3 = (int)(p % 3); p /= 3;
    const int xx = (int)(p % x.W); p /= x.W;
    const int yy = (int)(p % x.H);
    const int b = (int)(p / x.H);
    const float g = __half2float(tv(dout3, b, yy, xx)[k3 * x.C + c]);
    if (g == 0.f) continue;
    const int r = 2 + 2 * k3;   // radius 2 / 4 / 6
    float best = -INFINITY;
    int by = yy, bx = xx;
    for (int y2 = max(0, yy - r); y2 <= min(x.H - 1, yy + r); ++y2)
      for (int x2 = max(0, xx - r); x2 <= min(x.W - 1, xx + r); ++x2) {
        const float v = __half2float(tv(x, b, y2, x2)[c]);
        if (v > best) { best = v; by = y2; bx = x2; }
      }
    atomicAdd(scratch + (((size_t)b * x.H + by) * x.W + bx) * x.C + c, g);
  }
}
__global__ void add_scratch_kernel(TensorView dx, const float* scratch) {
  const long total = (long)dx.B * dx.H * dx.W * dx.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dx.C);
    const long p = i / dx.C;
    __half* d = reinterpret_cast<__half*>(dx.base) + (size_t)p * dx.ctot + c;
    *d = __float2half_rn(__half2float(*d) + scratch[i]);
  }
}
int launch_spp_bwd(const TensorView& x, const TensorView& dout3, const TensorView& dx, float* scratch, cudaStream_t s) {
  const long n = (long)x.B * x.H * x.W * x.C;
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (size_t)n * sizeof(float), s));
  spp_bwd_scatter_kernel<<<grid_for_t(n * 3, 128), 128, 0, s>>>(x, dout3, scratch);
  MYOLO_LAUNCH_CHECK();
  add_scratch_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(dx, scratch);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// adaptive pools: forward atoms = sum over cell, bins = sum(atoms)/count.
__global__ void region_combine_bwd_kernel(TensorView dbins, TensorView datoms, const int* __restrict__ bins, int nbins) {
  const long total = (long)dbins.B * nbins * dbins.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dbins.C);
    const int bin = (int)((i / dbins.C) % nbins);
    const int b = (int)(i / ((long)dbins.C * nbins));
    const int* bd = bins + bin * 5;
    const float g = ldv(dbins, b, bin / dbins.W, bin % dbins.W, c) / (float)bd[4];
    for (int ay = bd[0]; ay < bd[1]; ++ay)
      for (int ax = bd[2]; ax < bd[3]; ++ax) atomicAdd(tvf(datoms, b, ay, ax) + c, g);   // bins of one level are disjoint, levels are separate launches
  }
}
int launch_region_combine_bwd(const TensorView& dbins, const TensorView& datoms, int atoms_nx, const int* d_bins, int nbins, cudaStream_t s) {
  MYOLO_REQUIRE(datoms.dtype == MYOLO_F32, "region_combine_bwd: atoms gradient must be fp32");
  region_combine_bwd_kernel<<<grid_for_t((long)dbins.B * nbins * dbins.C, 256), 256, 0, s>>>(dbins, datoms, d_bins, nbins);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
__global__ void region_bwd_kernel(TensorView datoms, TensorView dx, const int* __restrict__ yb, int ny, const int* __restrict__ xb, int nx) {
  const long total = (long)dx.B * dx.H * dx.W * dx.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dx.C);
    long p = i / dx.C;
    const int x = (int)(p % dx.W); p /= dx.W;
    const int y = (int)(p % dx.H);
    const int b = (int)(p / dx.H);
    int ay = 0, ax = 0;
    while (ay + 1 < ny && y >= yb[ay + 1]) ++ay;
    while (ax + 1 < nx && x >= xb[ax + 1]) ++ax;
    stv(dx, b, y, x, c, ldv(dx, b, y, x, c) + tvf(datoms, b, ay, ax)[c]);
  }
}
int launch_region_bwd(const TensorView& datoms, const TensorView& dx, const int* d_yb, int ny, const int* d_xb, int nx, cudaStream_t s) {
  region_bwd_kernel<<<grid_for_t((long)dx.B * dx.H * dx.W * dx.C, 256), 256, 0, s>>>(datoms, dx, d_yb, ny, d_xb, nx);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void seg_upsample_bwd_kernel(const float* __restrict__ dseg, int ncls, int H, int W, TensorView dlo) {
  const long total = (long)dlo.B * dlo.H * dlo.W * ncls;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ncls);
    long p = i / ncls;
    const int x = (int)(p % dlo.W); p /= dlo.W;
    const int y = (int)(p % dlo.H);
    const int b = (int)(p / dlo.H);
    int ylo, yhi, xlo, xhi;
    dst_range(y, dlo.H, H, &ylo, &yhi);
    dst_range(x, dlo.W, W, &xlo, &xhi);
    const float* plane = dseg + ((size_t)b * ncls + c) * H * W;
    float acc = 0.f;
    for (int dy = ylo; dy <= yhi; ++dy) {
      int a0, a1; float w0, w1;
      lerp_src(dy, dlo.H, H, &a0, &a1, &w0, &w1);
      const float wy = (a0 == y ? w0 : 0.f) + (a1 == y ? w1 : 0.f);
      if (wy == 0.f) continue;
      for (int dx = xlo; dx <= xhi; ++dx) {
        int b0, b1; float v0, v1;
        lerp_src(dx, dlo.W, W, &b0, &b1, &v0, &v1);
        const float wx = (b0 == x ? v0 : 0.f) + (b1 == x ? v1 : 0.f);
        if (wx != 0.f) acc += wy * wx * plane[(size_t)dy * W + dx];
      }
    }
    tvf(dlo, b, y, x)[c] += acc;
  }
}
int launch_seg_upsample_bwd(const float* dseg, int n_cls, int H, int W, const TensorView& dlo, cudaStream_t s) {
  MYOLO_REQUIRE(dlo.dtype == MYOLO_F32, "seg_upsample_bwd: low-res logits gradient must be fp32");
  seg_upsample_bwd_kernel<<<grid_for_t((long)dlo.B * dlo.H * dlo.W * n_cls, 128), 128, 0, s>>>(dseg, n_cls, H, W, dlo);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Fused segmentation loss (SURVEY.md section 8f rank 3): CrossEntropyLoss(ignore_index) of the x8 bilinear (align_corners=True) upsample
// of the low-resolution logits, forward AND backward, without materialising the (B,C,H,W) logits or their gradient
// (reference models/yolo.py:163 + utils/loss.py:237 + autograd).  Thread = (low-res pixel, chunk of its footprint rows): every
// full-resolution pixel that reads this low-res pixel is revisited, its interpolated logits and softmax are recomputed from the 4
// low-res neighbours, and (p - onehot) * weight is accumulated; the thread that owns the pixel's top-left neighbour adds its loss.
//   dlo[b,y,x,c] += coef * sum_{(Y,X) reading (y,x)} w(Y,X;y,x) * (softmax_c(z(Y,X)) - [c == t(Y,X)]),   coef = factor * scale / n_valid
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}

// labels outside [0, n_cls) other than ignore_index would make torch's CrossEntropyLoss raise; here they count as ignored pixels
// (no device-side exception exists on this path; the python wrapper documents it)
__global__ void count_valid_kernel(const long long* __restrict__ labels, long n, int ignore_index, int n_cls, unsigned long long* out) {
  unsigned int c = 0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = labels[i];
    c += (t != ignore_index) && t >= 0 && t < n_cls;
  }
  c = __reduce_add_sync(0xFFFFFFFFu, c);
  if ((threadIdx.x & 31) == 0 && c) atomicAdd(out, (unsigned long long)c);
}

// ------------------------------------------------------------------------------------------------
// OHEM selection (reference utils/loss.py:321-328 OhemCELoss.forward_once) over a per-pixel CE buffer of n values, on the device and
// without a host synchronisation.  With n_min = n_valid // 16 and hard = #{loss > thresh_t}:
//   hard >= n_min: the hard pixels, mean over `hard` (hard == 0 gives 0/0 = NaN and no gradient, as torch.mean of an empty tensor);
//   otherwise:     the n_min largest losses (ignored pixels take part with loss 0), mean over n_min.  Among the pixels equal to the
//                  n_min-th largest value the lowest flat indices are taken (torch.topk leaves that order unspecified).
// The k-th largest value is a radix select over order-preserving 32-bit keys: four 8-bit histogram passes, each followed by a one-block
// digit pick.  Every kernel is always launched; kernels the batch's branch does not need return after reading `branch`, so one captured
// graph serves both branches.  A non-finite per-pixel loss makes the loss and every taken gradient NaN (GradScaler then skips the step).
// ------------------------------------------------------------------------------------------------
enum { kOhemThresh = 1, kOhemTopk = 2, kOhemNonFinite = 3 };
constexpr int kOhemChunk = 4096;           // pixels per block of the tie count; the cut kernel walks one chunk with 256 x 16 pixels

struct OhemSel {                           // zeroed before every selection
  unsigned int hist[4][256];
  unsigned long long n_valid;              // standalone loss: count_valid_kernel's output
  unsigned int hard, nonfinite;
  float hard_sum, gt_sum, thresh_t;
  int branch;
  unsigned int prefix;                     // after the four passes: the key of the n_min-th largest loss
  unsigned int k_rem;                      // pixels still to take among those matching `prefix`
  unsigned int tie_total;                  // pixels whose key equals the final prefix
  long long cut;                           // the highest flat index taken among the tied pixels
  float denom, loss_sum;
};

__device__ __forceinline__ unsigned ohem_key(float v) {
  unsigned u = __float_as_uint(v);
  if (u == 0x80000000u) u = 0u;                                   // -0.0 == +0.0: one key
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float ohem_key_value(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}
__device__ __forceinline__ bool ohem_taken(int branch, float thresh_t, unsigned kth, long long cut, long i, float v) {
  if (branch == kOhemThresh) return v > thresh_t;
  if (branch == kOhemTopk) {
    const unsigned k = ohem_key(v);
    return k > kth || (k == kth && i <= cut);
  }
  return branch == kOhemNonFinite;
}
__device__ __forceinline__ float ohem_coef(const OhemSel* st, float num) { return st->denom == 0.f ? 0.f : num / st->denom; }

// inclusive prefix sum over a 256-thread block; sh: 8 words of shared memory
__device__ unsigned block_scan256(unsigned v, unsigned* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned u = __shfl_up_sync(0xFFFFFFFFu, v, o);
    if (lane >= o) v += u;
  }
  if (lane == 31) sh[w] = v;
  __syncthreads();
  for (int i = 0; i < w; ++i) v += sh[i];
  __syncthreads();
  return v;
}

// pass p: histogram of key digit (31-8p .. 24-8p) over the pixels whose higher digits match the prefix; pass 0 also counts the hard pixels
__global__ void __launch_bounds__(256) ohem_hist_kernel(const float* __restrict__ loss, long n, OhemSel* st, int pass, float thresh_t) {
  if (pass > 0 && st->branch != kOhemTopk) return;
  __shared__ unsigned cnt[256];
  cnt[threadIdx.x] = 0;
  __syncthreads();
  const int shift = 24 - 8 * pass;
  const unsigned mask = pass ? 0xFFFFFFFFu << (32 - 8 * pass) : 0u, prefix = pass ? st->prefix : 0u;
  unsigned hard = 0, bad = 0;
  float hsum = 0.f;
  for (long base = (long)blockIdx.x * blockDim.x; base < n; base += (long)gridDim.x * blockDim.x) {    // warp-uniform trip count
    const long i = base + threadIdx.x;
    const float v = i < n ? loss[i] : 0.f;
    const unsigned k = ohem_key(v);
    const int d = (i < n && (k & mask) == prefix) ? (int)((k >> shift) & 255u) : 256;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, d);
    if (d < 256 && (int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&cnt[d], (unsigned)__popc(peers));
    if (pass == 0 && i < n) {
      if (v > thresh_t) { ++hard; hsum += v; }
      bad |= !isfinite(v);
    }
  }
  if (pass == 0) {
    hard = __reduce_add_sync(0xFFFFFFFFu, hard);
    bad = __reduce_or_sync(0xFFFFFFFFu, bad);
    hsum = warp_sum(hsum);
    if ((threadIdx.x & 31) == 0) {
      if (hard) { atomicAdd(&st->hard, hard); atomicAdd(&st->hard_sum, hsum); }
      if (bad) atomicOr(&st->nonfinite, 1u);
    }
  }
  __syncthreads();
  if (cnt[threadIdx.x]) atomicAdd(&st->hist[pass][threadIdx.x], cnt[threadIdx.x]);
}

// one block: pass 0 decides the branch; every pass of the top-k branch then picks the digit of the k-th largest key
__global__ void __launch_bounds__(256) ohem_pick_kernel(OhemSel* st, const unsigned long long* __restrict__ n_valid, int pass, float thresh_t) {
  __shared__ unsigned sh[8];
  unsigned k, prefix;
  if (pass == 0) {
    const unsigned long long n_min = *n_valid / 16;
    const unsigned hard = st->hard;
    int branch = kOhemTopk;
    if (st->nonfinite) branch = kOhemNonFinite;
    else if (hard >= n_min) branch = kOhemThresh;
    if (threadIdx.x == 0) {
      st->branch = branch;
      st->thresh_t = thresh_t;
      st->denom = branch == kOhemNonFinite ? NAN : branch == kOhemThresh ? (float)hard : (float)n_min;
      st->loss_sum = branch == kOhemNonFinite ? NAN : st->hard_sum;     // the top-k sum is written by ohem_cut_kernel
    }
    if (branch != kOhemTopk) return;
    k = (unsigned)n_min;
    prefix = 0u;
  } else {
    if (st->branch != kOhemTopk) return;
    k = st->k_rem;
    prefix = st->prefix;
  }
  const int d = 255 - (int)threadIdx.x;                                 // digits in descending order
  const unsigned c = st->hist[pass][d];
  const unsigned incl = block_scan256(c, sh);
  if (incl >= k && incl - c < k) {                                       // exactly one thread: k >= 1 and the digits hold >= k keys
    st->prefix = prefix | (unsigned)d << (24 - 8 * pass);
    st->k_rem = k - (incl - c);
    if (pass == 3) st->tie_total = c;
  }
}

// top-k branch: per chunk, the pixels tied at the k-th key; and the sum of the losses above it
__global__ void __launch_bounds__(256) ohem_tie_kernel(const float* __restrict__ loss, long n, OhemSel* st, unsigned* __restrict__ chunk_ties) {
  if (st->branch != kOhemTopk) return;
  __shared__ unsigned sh[8];
  const unsigned kth = st->prefix;
  const long lo = (long)blockIdx.x * kOhemChunk, hi = min(n, lo + kOhemChunk);
  unsigned ties = 0;
  float s = 0.f;
  for (long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const float v = loss[i];
    const unsigned k = ohem_key(v);
    ties += k == kth;
    if (k > kth) s += v;
  }
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0 && s != 0.f) atomicAdd(&st->gt_sum, s);
  ties = block_scan256(ties, sh);
  if (threadIdx.x == 255) chunk_ties[blockIdx.x] = ties;
}

// top-k branch, one block: the loss sum, and the index cutoff among the tied pixels when fewer than all of them are taken
__global__ void __launch_bounds__(256) ohem_cut_kernel(const float* __restrict__ loss, long n, OhemSel* st, const unsigned* __restrict__ chunk_ties,
                                                       int n_chunks) {
  if (st->branch != kOhemTopk) return;
  __shared__ unsigned sh[8];
  __shared__ int s_chunk;
  __shared__ unsigned s_r, s_total;
  const unsigned kth = st->prefix, need = st->k_rem;
  if (threadIdx.x == 0) {
    st->loss_sum = st->gt_sum + (float)need * ohem_key_value(kth);
    st->cut = LLONG_MAX;
    s_chunk = -1;
  }
  if (st->tie_total == need) return;
  __syncthreads();
  // the chunk holding the need-th tied pixel, then that pixel within it
  unsigned before = 0;
  for (int c0 = 0; c0 < n_chunks; c0 += 256) {
    const unsigned c = c0 + (int)threadIdx.x < n_chunks ? chunk_ties[c0 + threadIdx.x] : 0u;
    const unsigned incl = before + block_scan256(c, sh);
    if (c && incl >= need && incl - c < need) { s_chunk = c0 + threadIdx.x; s_r = need - (incl - c); }
    if (threadIdx.x == 255) s_total = incl;
    __syncthreads();
    if (s_chunk >= 0) break;
    before = s_total;
    __syncthreads();
  }
  if (s_chunk < 0) return;                 // unreachable: the chunk counts add up to tie_total > need
  const long lo = (long)s_chunk * kOhemChunk + threadIdx.x * (kOhemChunk / 256), hi = min(n, lo + kOhemChunk / 256);
  unsigned c = 0;
  for (long i = lo; i < hi; ++i) c += ohem_key(loss[i]) == kth;
  const unsigned incl = block_scan256(c, sh), r = s_r;
  if (c && incl >= r && incl - c < r) {
    unsigned left = r - (incl - c);
    for (long i = lo; i < hi; ++i)
      if (ohem_key(loss[i]) == kth && --left == 0) { st->cut = i; break; }
  }
}

static int ohem_select(const float* loss, long n, const unsigned long long* n_valid, float thresh_t, OhemSel* st, unsigned* chunk_ties,
                       cudaStream_t s) {
  const int n_chunks = (int)((n + kOhemChunk - 1) / kOhemChunk);
  for (int pass = 0; pass < 4; ++pass) {
    ohem_hist_kernel<<<grid_for_t(n, 256, 132 * 4), 256, 0, s>>>(loss, n, st, pass, thresh_t);
    MYOLO_LAUNCH_CHECK();
    ohem_pick_kernel<<<1, 256, 0, s>>>(st, n_valid, pass, thresh_t);
    MYOLO_LAUNCH_CHECK();
  }
  ohem_tie_kernel<<<n_chunks, 256, 0, s>>>(loss, n, st, chunk_ties);
  MYOLO_LAUNCH_CHECK();
  ohem_cut_kernel<<<1, 256, 0, s>>>(loss, n, st, chunk_ties, n_chunks);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

static size_t align256(size_t b) { return (b + 255) / 256 * 256; }
// workspace: [OhemSel][per-chunk tie counts][per-pixel loss, n floats]
size_t ohem_scratch_bytes(long n) {
  return align256(sizeof(OhemSel)) + align256((size_t)((n + kOhemChunk - 1) / kOhemChunk) * sizeof(unsigned)) + (size_t)n * sizeof(float);
}
struct OhemScratch {
  OhemSel* st;
  unsigned* ties;
  float* loss;
  size_t head;                             // bytes before the loss buffer (zeroed per call)
};
static OhemScratch ohem_scratch(void* ws, long n) {
  unsigned char* p = reinterpret_cast<unsigned char*>(ws);
  const size_t a = align256(sizeof(OhemSel)), b = align256((size_t)((n + kOhemChunk - 1) / kOhemChunk) * sizeof(unsigned));
  return {reinterpret_cast<OhemSel*>(p), reinterpret_cast<unsigned*>(p + a), reinterpret_cast<float*>(p + a + b), a + b};
}

__global__ void ohem_finalize_kernel(const OhemSel* st, float* loss_out) {
  if (loss_out) *loss_out = st->loss_sum / st->denom;
}

// ------------------------------------------------------------------------------------------------
// Class-weighted CE and focal loss (reference SegmentationLosses(weight=w), utils/loss.py:221-237, and SegFocalLoss, :279-297).  With
// t' = t for valid pixels and 0 for ignored ones (the reference's `target * (target != ignore_index)`), p = softmax(z), N pixels:
//   A = sum_valid w[t] CE / sum_valid w[t]  (mean)  or  sum_valid w[t] CE  (sum)         the CE inside SegFocalLoss takes its reduction
//   F = sum_all (1 - p_t')^gamma / N        (mean)  or  sum_all (1 - p_t')^gamma (sum)   ignored pixels take part, with class 0
//   loss = A * F;   d loss / d z_i = (c1 * w[t_i] [valid_i] + c2 * gamma (1 - p_t')^(gamma-1) p_t') * (p_i - e_t')
// with c1 = F / sum w (mean) or F (sum), c2 = A / N (mean) or A (sum).  gamma = 0 is the weighted CE: F = 1 (or N) exactly and c2 = 0,
// as torch's pow backward returns zeros for a zero exponent.  Three sums over the pixels, then one finalize thread writes the loss and
// the coefficients; nothing returns to the host.  Null weights are unit weights.  No valid pixel gives A = 0 / 0 = NaN, and the gradient
// is NaN with gamma > 0 (A enters every pixel's gradient) and zero with gamma = 0, as in the reference.
// ------------------------------------------------------------------------------------------------
struct SegWfSt {
  float s_wl, s_w, s_f;                    // zeroed per call: sum_valid w[t] CE, sum_valid w[t], sum_all (1 - p_t')^gamma
  float c1, c2, loss;
};
constexpr size_t kSegWfHead = 256;         // the SegWfSt, padded; the fused pass's per-pixel factors follow it

__device__ __forceinline__ float focal_grad_factor(float pt, float gamma) {
  return gamma == 0.f ? 0.f : gamma * powf(1.f - pt, gamma - 1.f) * pt;   // p_t' = 1 with gamma < 1: inf, as torch's pow backward
}

__device__ __forceinline__ void seg_wf_accumulate(SegWfSt* st, float swl, float sw, float sf) {
  swl = warp_sum(swl); sw = warp_sum(sw); sf = warp_sum(sf);
  if ((threadIdx.x & 31) == 0) {
    if (sw != 0.f || swl != 0.f) { atomicAdd(&st->s_wl, swl); atomicAdd(&st->s_w, sw); }
    if (sf != 0.f) atomicAdd(&st->s_f, sf);
  }
}

__global__ void seg_wf_finalize_kernel(SegWfSt* st, float gamma, float n, int sum, float* loss_out) {
  const float A = sum ? st->s_wl : st->s_wl / st->s_w;
  const float F = gamma == 0.f ? (sum ? n : 1.f) : (sum ? st->s_f : st->s_f / n);
  st->c1 = sum ? F : (st->s_w == 0.f ? 0.f : F / st->s_w);
  st->c2 = gamma == 0.f ? 0.f : (sum ? A : A / n);
  st->loss = A * F;
  if (loss_out) *loss_out = st->loss;
}

// the weighted / focal mode of the fused pass: per-class weights (nullable), gamma, and per pixel the two factors
// (w[t] [valid], gamma (1 - p_t')^(gamma-1) p_t') the gather combines with the finalized c1, c2
struct SegWf {
  const float* w;
  float gamma;
  SegWfSt* st;
  float2* pf;
};

// pass 1: one thread per FULL-resolution pixel: interpolated logits from the 4 low-res neighbours -> softmax -> (p - onehot) written as
// NC_PAD fp32 per pixel (zeros for ignored pixels); the pixel's loss is reduced per warp, and written to pix_loss (OHEM, nullable).
template <int NC, int NC_PAD>
__global__ void seg_ce_pixel_kernel(TensorView lo, const long long* __restrict__ labels, int H, int W, int ignore_index, float* __restrict__ g,
                                    float* loss_sum, float* __restrict__ pix_loss) {
  const long total = (long)lo.B * H * W;
  float loss_local = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const int b = (int)(i / ((long)W * H));
    const long long t = labels[i];
    float v[NC_PAD], l = 0.f;
#pragma unroll
    for (int c = 0; c < NC_PAD; ++c) v[c] = 0.f;
    if (t != ignore_index && t >= 0 && t < NC) {
      int a0, a1, b0, b1; float w0, w1, v0, v1;
      lerp_src(Y, lo.H, H, &a0, &a1, &w0, &w1);
      lerp_src(X, lo.W, W, &b0, &b1, &v0, &v1);
      const float* q00 = tvf(lo, b, a0, b0); const float* q01 = tvf(lo, b, a0, b1);
      const float* q10 = tvf(lo, b, a1, b0); const float* q11 = tvf(lo, b, a1, b1);
      const float c00 = w0 * v0, c01 = w0 * v1, c10 = w1 * v0, c11 = w1 * v1;
      float m = -INFINITY, zt = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) { v[c] = c00 * q00[c] + c01 * q01[c] + c10 * q10[c] + c11 * q11[c]; m = fmaxf(m, v[c]); }
      float ssum = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) { if (c == (int)t) zt = v[c]; v[c] = __expf(v[c] - m); ssum += v[c]; }
      const float inv = 1.0f / ssum;
#pragma unroll
      for (int c = 0; c < NC; ++c) v[c] = v[c] * inv - (c == (int)t ? 1.0f : 0.f);
      l = __logf(ssum) + m - zt;
      loss_local += l;
    }
    if (pix_loss) pix_loss[i] = l;
    float4* dst = reinterpret_cast<float4*>(g + (size_t)i * NC_PAD);
#pragma unroll
    for (int c = 0; c < NC_PAD; c += 4) dst[c / 4] = make_float4(v[c], v[c + 1], v[c + 2], v[c + 3]);
  }
  loss_local = warp_sum(loss_local);
  if ((threadIdx.x & 31) == 0 && loss_local != 0.f) atomicAdd(loss_sum, loss_local);
}

// pass 1 of the weighted / focal loss: seg_ce_pixel_kernel's per-pixel (p - onehot(t')), and the pixel's two factors (w[t] [valid],
// gamma (1 - p_t')^(gamma-1) p_t') for the gather; the three sums are reduced per warp.  With gamma != 0 the ignored pixels' softmax is
// taken too, against class 0.
template <int NC, int NC_PAD>
__global__ void seg_wf_pixel_kernel(TensorView lo, const long long* __restrict__ labels, int H, int W, int ignore_index, float* __restrict__ g,
                                    SegWf wf) {
  const long total = (long)lo.B * H * W;
  float swl = 0.f, sw = 0.f, sf = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const int b = (int)(i / ((long)W * H));
    const long long t = labels[i];
    const bool valid = t != ignore_index && t >= 0 && t < NC;
    const int tt = valid ? (int)t : 0;
    float v[NC_PAD];
    float2 f = make_float2(0.f, 0.f);
#pragma unroll
    for (int c = 0; c < NC_PAD; ++c) v[c] = 0.f;
    if (valid || wf.gamma != 0.f) {
      int a0, a1, b0, b1; float w0, w1, v0, v1;
      lerp_src(Y, lo.H, H, &a0, &a1, &w0, &w1);
      lerp_src(X, lo.W, W, &b0, &b1, &v0, &v1);
      const float* q00 = tvf(lo, b, a0, b0); const float* q01 = tvf(lo, b, a0, b1);
      const float* q10 = tvf(lo, b, a1, b0); const float* q11 = tvf(lo, b, a1, b1);
      const float c00 = w0 * v0, c01 = w0 * v1, c10 = w1 * v0, c11 = w1 * v1;
      float m = -INFINITY, zt = 0.f, et = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) { v[c] = c00 * q00[c] + c01 * q01[c] + c10 * q10[c] + c11 * q11[c]; m = fmaxf(m, v[c]); }
      float ssum = 0.f;
#pragma unroll
      for (int c = 0; c < NC; ++c) { if (c == tt) zt = v[c]; v[c] = __expf(v[c] - m); if (c == tt) et = v[c]; ssum += v[c]; }
      const float inv = 1.0f / ssum;
#pragma unroll
      for (int c = 0; c < NC; ++c) v[c] = v[c] * inv - (c == tt ? 1.0f : 0.f);
      const float pt = et * inv;
      if (valid) {
        f.x = wf.w ? wf.w[tt] : 1.f;
        swl += f.x * (__logf(ssum) + m - zt);
        sw += f.x;
      }
      if (wf.gamma != 0.f) {
        f.y = focal_grad_factor(pt, wf.gamma);
        sf += powf(1.f - pt, wf.gamma);
      }
    }
    wf.pf[i] = f;
    float4* dst = reinterpret_cast<float4*>(g + (size_t)i * NC_PAD);
#pragma unroll
    for (int c = 0; c < NC_PAD; c += 4) dst[c / 4] = make_float4(v[c], v[c + 1], v[c + 2], v[c + 3]);
  }
  seg_wf_accumulate(wf.st, swl, sw, sf);
}

// pass 2: adjoint of the bilinear upsample, gathered per low-res pixel (x a chunk of its footprint rows) from the per-pixel gradients.
// OHEM (sel non-null): only the pixels the selection took contribute, and the denominator is the selection's.
// WF: each pixel's gradient is scaled by c1 * pf.x + c2 * pf.y (seg_wf_finalize_kernel).
template <int NC, int NC_PAD, bool WF>
__global__ void seg_ce_gather_kernel(const float* __restrict__ g, int H, int W, TensorView dlo, float factor, const float* __restrict__ scale_dev,
                                     const unsigned long long* __restrict__ n_valid, int rsplit, const OhemSel* __restrict__ sel,
                                     const float* __restrict__ pix_loss, const SegWfSt* __restrict__ wst, const float2* __restrict__ pf) {
  const long total = (long)dlo.B * dlo.H * dlo.W * rsplit;
  const float num = factor * (scale_dev ? *scale_dev : 1.0f);
  float coef;
  int branch = 0;
  float thresh_t = 0.f;
  unsigned kth = 0;
  long long cut = 0;
  float c1 = 0.f, c2 = 0.f;
  if constexpr (WF) {
    coef = num;
    c1 = wst->c1; c2 = wst->c2;
  } else if (sel) {
    coef = ohem_coef(sel, num);
    branch = sel->branch; thresh_t = sel->thresh_t; kth = sel->prefix; cut = sel->cut;
  } else {
    const unsigned long long nv = *n_valid;
    coef = nv ? num / (float)nv : 0.f;
  }
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int part = (int)(i % rsplit);
    long p = i / rsplit;
    const int x = (int)(p % dlo.W); p /= dlo.W;
    const int y = (int)(p % dlo.H);
    const int b = (int)(p / dlo.H);
    int ylo, yhi, xlo, xhi;
    dst_range(y, dlo.H, H, &ylo, &yhi);
    dst_range(x, dlo.W, W, &xlo, &xhi);
    const int rows = yhi - ylo + 1, per = (rows + rsplit - 1) / rsplit;
    const int r0 = ylo + part * per, r1 = min(yhi, r0 + per - 1);
    float acc[NC_PAD];
#pragma unroll
    for (int c = 0; c < NC_PAD; ++c) acc[c] = 0.f;
    for (int Y = r0; Y <= r1; ++Y) {
      int a0, a1; float w0, w1;
      lerp_src(Y, dlo.H, H, &a0, &a1, &w0, &w1);
      const float wy = (a0 == y ? w0 : 0.f) + (a1 == y ? w1 : 0.f);
      if (wy == 0.f) continue;
      const float* row = g + ((size_t)b * H + Y) * W * NC_PAD;
      for (int X = xlo; X <= xhi; ++X) {
        int b0, b1; float v0, v1;
        lerp_src(X, dlo.W, W, &b0, &b1, &v0, &v1);
        float wgt = wy * ((b0 == x ? v0 : 0.f) + (b1 == x ? v1 : 0.f));
        if (wgt == 0.f) continue;
        if constexpr (WF) {
          const float2 f = pf[((long)b * H + Y) * W + X];
          const float k = c1 * f.x + c2 * f.y;
          if (k == 0.f) continue;
          wgt *= k;
        } else if (sel) {
          const long pix = ((long)b * H + Y) * W + X;
          if (!ohem_taken(branch, thresh_t, kth, cut, pix, pix_loss[pix])) continue;
        }
        const float4* q = reinterpret_cast<const float4*>(row + (size_t)X * NC_PAD);
#pragma unroll
        for (int c = 0; c < NC_PAD; c += 4) {
          const float4 u = q[c / 4];
          acc[c] += wgt * u.x; acc[c + 1] += wgt * u.y; acc[c + 2] += wgt * u.z; acc[c + 3] += wgt * u.w;
        }
      }
    }
    float* d = tvf(dlo, b, y, x);
#pragma unroll
    for (int c = 0; c < NC; ++c)
      if (acc[c] != 0.f) atomicAdd(d + c, acc[c] * coef);
  }
}

__global__ void seg_ce_finalize_kernel(const float* loss_sum, const unsigned long long* n_valid, float* loss_out) {
  if (loss_out) *loss_out = *n_valid ? *loss_sum / (float)*n_valid : 0.f;     // mean over the valid pixels (F.cross_entropy)
}

size_t seg_ce_scratch_bytes(int B, int H, int W, int n_cls) { return (size_t)B * H * W * (n_cls <= 20 ? 20 : 32) * sizeof(float); }

// scratch16: 16 bytes (n_valid u64, loss_sum f32); gbuf: seg_ce_scratch_bytes.  loss_out (device, nullable) receives the mean CE.
// ohem_ws (nullable): ohem_scratch_bytes(B*H*W) bytes; the loss becomes OhemCELoss(thresh) with thresh_t = -log(thresh).
int launch_seg_ce_fused(const TensorView& lo, int n_cls, const long long* labels, int H, int W, int ignore_index, const TensorView& dlo,
                        float factor, const float* scale_dev, void* scratch16, float* gbuf, float* loss_out, cudaStream_t s, void* ohem_ws,
                        float thresh_t) {
  MYOLO_REQUIRE(lo.dtype == MYOLO_F32 && dlo.dtype == MYOLO_F32 && n_cls >= 1 && n_cls <= 32 && lo.C >= n_cls && labels && scratch16 && gbuf,
                "seg_ce_fused: fp32 low-resolution logits with <= 32 classes expected");
  MYOLO_REQUIRE(n_cls == 19 || n_cls == 32, "seg_ce_fused: instantiate the kernels for %d classes (19 and 32 are built)", n_cls);
  unsigned long long* n_valid = reinterpret_cast<unsigned long long*>(scratch16);
  float* loss_sum = reinterpret_cast<float*>(n_valid + 1);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch16, 0, 16, s));
  const long n = (long)lo.B * H * W;
  OhemScratch oh{nullptr, nullptr, nullptr, 0};
  if (ohem_ws) {
    oh = ohem_scratch(ohem_ws, n);
    MYOLO_CHECK_CUDA(cudaMemsetAsync(ohem_ws, 0, oh.head, s));
  }
  count_valid_kernel<<<grid_for_t(n, 256, 132 * 8), 256, 0, s>>>(labels, n, ignore_index, n_cls, n_valid);
  MYOLO_LAUNCH_CHECK();
  const int rsplit = 4;
  const int g1 = grid_for_t(n, 128), g2 = grid_for_t((long)lo.B * lo.H * lo.W * rsplit, 128);
  if (n_cls == 19) seg_ce_pixel_kernel<19, 20><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, loss_sum, oh.loss);
  else seg_ce_pixel_kernel<32, 32><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, loss_sum, oh.loss);
  MYOLO_LAUNCH_CHECK();
  if (ohem_ws)
    if (int rc = ohem_select(oh.loss, n, n_valid, thresh_t, oh.st, oh.ties, s)) return rc;
  if (n_cls == 19)
    seg_ce_gather_kernel<19, 20, false><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, n_valid, rsplit, oh.st, oh.loss, nullptr, nullptr);
  else
    seg_ce_gather_kernel<32, 32, false><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, n_valid, rsplit, oh.st, oh.loss, nullptr, nullptr);
  MYOLO_LAUNCH_CHECK();
  if (ohem_ws) ohem_finalize_kernel<<<1, 1, 0, s>>>(oh.st, loss_out);
  else seg_ce_finalize_kernel<<<1, 1, 0, s>>>(loss_sum, n_valid, loss_out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

size_t seg_wf_scratch_bytes(long n) { return kSegWfHead + (size_t)n * sizeof(float2); }

// the weighted / focal loss in place of the mean CE: wf_ws = seg_wf_scratch_bytes(B*H*W) bytes; weights: n_cls device floats (nullable)
int launch_seg_wf_fused(const TensorView& lo, int n_cls, const long long* labels, int H, int W, int ignore_index, const TensorView& dlo,
                        float factor, const float* scale_dev, float* gbuf, void* wf_ws, const float* weights, float gamma, float* loss_out,
                        cudaStream_t s) {
  MYOLO_REQUIRE(lo.dtype == MYOLO_F32 && dlo.dtype == MYOLO_F32 && lo.C >= n_cls && labels && gbuf && wf_ws,
                "seg_loss_fused: fp32 low-resolution logits expected");
  MYOLO_REQUIRE(n_cls == 19 || n_cls == 32, "seg_loss_fused: instantiate the kernels for %d classes (19 and 32 are built)", n_cls);
  MYOLO_REQUIRE(gamma >= 0.f && isfinite(gamma), "seg_loss_fused: gamma must be finite and >= 0, got %g", (double)gamma);
  const long n = (long)lo.B * H * W;
  SegWf wf{weights, gamma, reinterpret_cast<SegWfSt*>(wf_ws), reinterpret_cast<float2*>(reinterpret_cast<unsigned char*>(wf_ws) + kSegWfHead)};
  MYOLO_CHECK_CUDA(cudaMemsetAsync(wf_ws, 0, sizeof(SegWfSt), s));
  const int rsplit = 4;
  const int g1 = grid_for_t(n, 128), g2 = grid_for_t((long)lo.B * lo.H * lo.W * rsplit, 128);
  if (n_cls == 19) seg_wf_pixel_kernel<19, 20><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, wf);
  else seg_wf_pixel_kernel<32, 32><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, wf);
  MYOLO_LAUNCH_CHECK();
  seg_wf_finalize_kernel<<<1, 1, 0, s>>>(wf.st, gamma, (float)n, 0, loss_out);
  MYOLO_LAUNCH_CHECK();
  if (n_cls == 19)
    seg_ce_gather_kernel<19, 20, true><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, nullptr, rsplit, nullptr, nullptr, wf.st, wf.pf);
  else
    seg_ce_gather_kernel<32, 32, true><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, nullptr, rsplit, nullptr, nullptr, wf.st, wf.pf);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ---- SegFocalLoss over full-resolution NCHW fp32 logits of any class count (the standalone module: utils.loss.SegFocalLoss) ----
__global__ void seg_focal_nchw_kernel(const float* __restrict__ x, const long long* __restrict__ labels, int B, int C, long HW,
                                      int ignore_index, const float* __restrict__ w, float gamma, SegWfSt* st) {
  const long n = (long)B * HW;
  float swl = 0.f, sw = 0.f, sf = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = labels[i];
    const bool valid = t != ignore_index && t >= 0 && t < C;
    if (!valid && gamma == 0.f) continue;
    const int tt = valid ? (int)t : 0;
    const float* xp = x + (size_t)(i / HW) * C * HW + i % HW;
    float m = -INFINITY;
    for (int c = 0; c < C; ++c) m = fmaxf(m, xp[(size_t)c * HW]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(xp[(size_t)c * HW] - m);
    const float zt = xp[(size_t)tt * HW];
    if (valid) {
      const float a = w ? w[tt] : 1.f;
      swl += a * (logf(s) + m - zt);
      sw += a;
    }
    if (gamma != 0.f) sf += powf(1.f - expf(zt - m) / s, gamma);
  }
  seg_wf_accumulate(st, swl, sw, sf);
}

// dx = grad_out * (c1 * w[t] [valid] + c2 * gamma (1 - p_t')^(gamma-1) p_t') * (softmax - onehot(t'))
__global__ void seg_focal_nchw_bwd_kernel(const float* __restrict__ x, const long long* __restrict__ labels, int B, int C, long HW,
                                          int ignore_index, const float* __restrict__ w, float gamma, const SegWfSt* __restrict__ st,
                                          const float* __restrict__ grad_out, float* __restrict__ dx) {
  const long n = (long)B * HW;
  const float go = *grad_out, c1 = st->c1, c2 = st->c2;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = labels[i];
    const bool valid = t != ignore_index && t >= 0 && t < C;
    const int tt = valid ? (int)t : 0;
    const size_t base = (size_t)(i / HW) * C * HW + i % HW;
    const float* xp = x + base;
    float* dp = dx + base;
    float m = -INFINITY, s = 0.f, k = 0.f;
    if (valid || gamma != 0.f) {
      for (int c = 0; c < C; ++c) m = fmaxf(m, xp[(size_t)c * HW]);
      for (int c = 0; c < C; ++c) s += expf(xp[(size_t)c * HW] - m);
      const float a = valid ? (w ? w[tt] : 1.f) : 0.f;
      k = go * (c1 * a + c2 * focal_grad_factor(expf(xp[(size_t)tt * HW] - m) / s, gamma));
    }
    if (k == 0.f) {
      for (int c = 0; c < C; ++c) dp[(size_t)c * HW] = 0.f;
      continue;
    }
    const float inv = 1.0f / s;
    for (int c = 0; c < C; ++c) dp[(size_t)c * HW] = k * (expf(xp[(size_t)c * HW] - m) * inv - (c == tt ? 1.0f : 0.f));
  }
}

// ---- OhemCELoss over full-resolution NCHW fp32 logits of any class count (the standalone module: utils.loss.OhemCELoss) ----
__global__ void ohem_ce_nchw_kernel(const float* __restrict__ x, const long long* __restrict__ labels, int B, int C, long HW, int ignore_index,
                                    float* __restrict__ loss) {
  const long n = (long)B * HW;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = labels[i];
    float l = 0.f;
    if (t != ignore_index && t >= 0 && t < C) {
      const float* xp = x + (size_t)(i / HW) * C * HW + i % HW;
      float m = -INFINITY;
      for (int c = 0; c < C; ++c) m = fmaxf(m, xp[(size_t)c * HW]);
      float s = 0.f;
      for (int c = 0; c < C; ++c) s += expf(xp[(size_t)c * HW] - m);
      l = logf(s) + m - xp[(size_t)t * HW];
    }
    loss[i] = l;
  }
}

// dx = grad_out * taken * (softmax - onehot) / denominator; pixels the selection did not take get 0
__global__ void ohem_ce_nchw_bwd_kernel(const float* __restrict__ x, const long long* __restrict__ labels, int B, int C, long HW, int ignore_index,
                                        const float* __restrict__ pix_loss, const OhemSel* __restrict__ sel, const float* __restrict__ grad_out,
                                        float* __restrict__ dx) {
  const long n = (long)B * HW;
  const float coef = ohem_coef(sel, *grad_out);
  const int branch = sel->branch;
  const float thresh_t = sel->thresh_t;
  const unsigned kth = sel->prefix;
  const long long cut = sel->cut;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const long long t = labels[i];
    const size_t base = (size_t)(i / HW) * C * HW + i % HW;
    const float* xp = x + base;
    float* dp = dx + base;
    if (t == ignore_index || t < 0 || t >= C || !ohem_taken(branch, thresh_t, kth, cut, i, pix_loss[i])) {
      for (int c = 0; c < C; ++c) dp[(size_t)c * HW] = 0.f;
      continue;
    }
    float m = -INFINITY;
    for (int c = 0; c < C; ++c) m = fmaxf(m, xp[(size_t)c * HW]);
    float s = 0.f;
    for (int c = 0; c < C; ++c) s += expf(xp[(size_t)c * HW] - m);
    const float inv = 1.0f / s;
    for (int c = 0; c < C; ++c) dp[(size_t)c * HW] = coef * (expf(xp[(size_t)c * HW] - m) * inv - (c == (int)t ? 1.0f : 0.f));
  }
}

__global__ void detect_raw_bwd_kernel(const float* __restrict__ draw, int na, int no, TensorView dconv) {
  const long total = (long)dconv.B * na * dconv.H * dconv.W * no;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int o = (int)(i % no);
    long p = i / no;
    const int x = (int)(p % dconv.W); p /= dconv.W;
    const int y = (int)(p % dconv.H); p /= dconv.H;
    const int a = (int)(p % na);
    const int b = (int)(p / na);
    tvf(dconv, b, y, x)[a * no + o] += draw[i];
  }
}
int launch_detect_raw_bwd(const float* draw, int na, int no, const TensorView& dconv, cudaStream_t s) {
  MYOLO_REQUIRE(dconv.dtype == MYOLO_F32 && dconv.ctot >= na * no, "detect_raw_bwd: bad view");
  detect_raw_bwd_kernel<<<grid_for_t((long)dconv.B * na * dconv.H * dconv.W * no, 256), 256, 0, s>>>(draw, na, no, dconv);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void cast_kernel(TensorView src, TensorView dst, int acc) {
  const int C = min(src.C, dst.C);
  const long total = (long)dst.B * dst.H * dst.W * dst.C;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % dst.C);
    long p = i / dst.C;
    const int x = (int)(p % dst.W); p /= dst.W;
    const int y = (int)(p % dst.H);
    const int b = (int)(p / dst.H);
    const float v = c < C ? ldv(src, b, y, x, c) : 0.f;
    stv(dst, b, y, x, c, acc ? ldv(dst, b, y, x, c) + v : v);
  }
}
int launch_cast_f32_to_f16(const TensorView& src, const TensorView& dst, cudaStream_t s) {
  cast_kernel<<<grid_for_t((long)dst.B * dst.H * dst.W * dst.C, 256), 256, 0, s>>>(src, dst, 0);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
int launch_cast_f16_to_f32_acc(const TensorView& src, const TensorView& dst, cudaStream_t s) {
  cast_kernel<<<grid_for_t((long)dst.B * dst.H * dst.W * dst.C, 256), 256, 0, s>>>(src, dst, 1);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void zero_stuff2_kernel(TensorView src, TensorView dst) {
  const int nv = dst.C / 8;
  const long total = (long)dst.B * dst.H * dst.W * nv;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int v = (int)(i % nv);
    long p = i / nv;
    const int x = (int)(p % dst.W); p /= dst.W;
    const int y = (int)(p % dst.H);
    const int b = (int)(p / dst.H);
    uint4 val = make_uint4(0, 0, 0, 0);
    if (!(x & 1) && !(y & 1)) val = reinterpret_cast<const uint4*>(tv(src, b, y >> 1, x >> 1))[v];
    reinterpret_cast<uint4*>(tv(dst, b, y, x))[v] = val;
  }
}
int launch_zero_stuff2(const TensorView& src, const TensorView& dst, cudaStream_t s) {
  MYOLO_REQUIRE(dst.H == 2 * src.H && dst.W == 2 * src.W && dst.C == src.C && dst.C % 8 == 0 && src.ctot % 8 == 0 && dst.ctot % 8 == 0,
                "zero_stuff2: bad views");
  zero_stuff2_kernel<<<grid_for_t((long)dst.B * dst.H * dst.W * (dst.C / 8), 256), 256, 0, s>>>(src, dst);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// dgrad weights: W'[ci][tap'][co] = W[co][ci][k*k-1-tap']   (fp16, [Ci_pad_out][k*k][Co_pad_in]); zero bias of length Ci_pad_out
__global__ void pack_dgrad_kernel(const float* __restrict__ w, int co, int ci, int k, __half* wp, float* zb, int ci_pad_out, int co_pad_in) {
  // waits for its predecessor but does NOT release its dependents early: the data-gradient conv that may follow fetches these weights
  // BEFORE its own dependency wait (weights are constants for every other predecessor)
  asm volatile("griddepcontrol.wait;" ::: "memory");
  const int taps = k * k;
  const long total = (long)ci_pad_out * taps * co_pad_in;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int o = (int)(i % co_pad_in);
    const int t = (int)((i / co_pad_in) % taps);
    const int c = (int)(i / ((long)co_pad_in * taps));
    float v = 0.f;
    if (c < ci && o < co) v = w[((size_t)o * ci + c) * taps + (taps - 1 - t)];
    wp[i] = __float2half_rn(v);
  }
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < ci_pad_out; c += gridDim.x * blockDim.x) zb[c] = 0.f;
}
int pack_dgrad_weights(const float* w, int co, int ci, int k, __half* wp, float* zero_bias, int ci_pad_out, int co_pad_in, cudaStream_t s) {
  MYOLO_CHECK_CUDA(launch_pdl(pack_dgrad_kernel, dim3(grid_for_t((long)ci_pad_out * k * k * co_pad_in, 256, 4096)), dim3(256), 0, s, w, co, ci, k,
                              wp, zero_bias, ci_pad_out, co_pad_in));
  g_launch_count++;
  return 0;
}

// ------------------------------------------------------------------------------------------------
// weight gradient: dW[co][ci][tap] += sum over output pixels p of dY[p][co] * X[in(p, tap)][ci]
// one CTA = 64 co x 64 ci x one tap x one slab of pixels; mma.sync.m16n8k16 with ldmatrix.trans from [pixel][channel] smem tiles
// ------------------------------------------------------------------------------------------------
static constexpr int kWgPitch = 72;   // halves per smem row (64 + 8 pad): conflict-free 8x8 ldmatrix
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__global__ void __launch_bounds__(128) conv_wgrad_kernel(TensorView x, TensorView dy, int k, int stride, int dil, float* dW, int co, int ci,
                                                         int splits) {
  __shared__ __align__(16) __half s_dy[32 * kWgPitch];
  __shared__ __align__(16) __half s_x[32 * kWgPitch];
  const int taps = k * k;
  const int co0 = blockIdx.x * 64;
  const int ci_tiles = (ci + 63) / 64;
  const int ci0 = (blockIdx.y % ci_tiles) * 64, tap = blockIdx.y / ci_tiles;
  const int ky = tap / k, kx = tap % k, pad = dil * (k / 2);
  const long npix = (long)dy.B * dy.H * dy.W;
  const long chunks = (npix + 31) / 32;
  const long c_begin = chunks * blockIdx.z / splits, c_end = chunks * (blockIdx.z + 1) / splits;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wm = (warp >> 1) * 32, wn = (warp & 1) * 32;   // warp tile origin inside the 64 x 64 CTA tile
  float acc[2][4][4];
#pragma unroll
  for (int a = 0; a < 2; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[a][b][e] = 0.f;
  const uint32_t sdy = smem_u32(s_dy), sx = smem_u32(s_x);
  for (long ch = c_begin; ch < c_end; ++ch) {
    // stage 32 pixels: 8 x 16-byte units per row, 2 units per thread per matrix
    for (int u = threadIdx.x; u < 32 * 8; u += 128) {
      const int r = u >> 3, v = u & 7;
      const long p = ch * 32 + r;
      uint4 qd = make_uint4(0, 0, 0, 0), qx = make_uint4(0, 0, 0, 0);
      if (p < npix) {
        const int ox = (int)(p % dy.W);
        const int oy = (int)((p / dy.W) % dy.H);
        const int b = (int)(p / ((long)dy.W * dy.H));
        if (co0 + v * 8 < co) qd = *reinterpret_cast<const uint4*>(tv(dy, b, oy, ox) + co0 + v * 8);
        const int iy = oy * stride - pad + ky * dil, ix = ox * stride - pad + kx * dil;
        if (iy >= 0 && iy < x.H && ix >= 0 && ix < x.W && ci0 + v * 8 < ci) qx = *reinterpret_cast<const uint4*>(tv(x, b, iy, ix) + ci0 + v * 8);
      }
      *reinterpret_cast<uint4*>(s_dy + r * kWgPitch + v * 8) = qd;
      *reinterpret_cast<uint4*>(s_x + r * kWgPitch + v * 8) = qx;
    }
    __syncthreads();
#pragma unroll
    for (int k0 = 0; k0 < 32; k0 += 16) {
      uint32_t af[2][4], bf[4][2];
      // A(m = co, k = pixel) from s_dy[k][m] via .trans: matrices (k0,m0) (k0,m0+8) (k0+8,m0) (k0+8,m0+8)
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const int m0 = wm + mt * 16;
        const int row = k0 + (lane & 7) + ((lane >> 4) << 3), col = m0 + (((lane >> 3) & 1) << 3);
        ldsm_x4_trans(sdy + (row * kWgPitch + col) * 2, af[mt][0], af[mt][1], af[mt][2], af[mt][3]);
      }
      // B(k = pixel, n = ci) from s_x[k][n] via .trans: matrices (k0,n0) (k0+8,n0) (k0,n0+8) (k0+8,n0+8)
#pragma unroll
      for (int nt2 = 0; nt2 < 2; ++nt2) {
        const int n0 = wn + nt2 * 16;
        const int row = k0 + (lane & 7) + (((lane >> 3) & 1) << 3), col = n0 + ((lane >> 4) << 3);
        ldsm_x4_trans(sx + (row * kWgPitch + col) * 2, bf[2 * nt2][0], bf[2 * nt2][1], bf[2 * nt2 + 1][0], bf[2 * nt2 + 1][1]);
      }
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < 4; ++nt) mma16816(acc[mt][nt], af[mt][0], af[mt][1], af[mt][2], af[mt][3], bf[nt][0], bf[nt][1]);
    }
    __syncthreads();
  }
  // C fragment: rows g, g+8; cols 2t, 2t+1
  const int g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 4; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int o = co0 + wm + mt * 16 + g + ((e >> 1) << 3);
        const int c = ci0 + wn + nt * 8 + 2 * t + (e & 1);
        if (o < co && c < ci) atomicAdd(dW + ((size_t)o * ci + c) * taps + tap, acc[mt][nt][e]);
      }
}

int launch_conv_wgrad(const TensorView& x, const TensorView& dy, int k, int stride, int dil, float* dW, int co, int ci, float* dbias,
                      cudaStream_t s) {
  MYOLO_REQUIRE(x.dtype == MYOLO_F16 && dy.dtype == MYOLO_F16 && x.ctot % 8 == 0 && dy.ctot % 8 == 0, "conv_wgrad: fp16 NHWC views expected");
  MYOLO_REQUIRE(x.C >= ci && dy.C >= co, "conv_wgrad: views narrower than the weight (%d<%d or %d<%d)", x.C, ci, dy.C, co);
  const long npix = (long)dy.B * dy.H * dy.W;
  const int tiles = ceil_div(co, 64) * ceil_div(ci, 64) * k * k;
  long chunks = (npix + 31) / 32;
  int splits = (int)std::min<long>(chunks, std::max<long>(1, (132L * 8) / tiles));
  dim3 grid(ceil_div(co, 64), ceil_div(ci, 64) * k * k, splits);
  conv_wgrad_kernel<<<grid, 128, 0, s>>>(x, dy, k, stride, dil, dW, co, ci, splits);
  MYOLO_LAUNCH_CHECK();
  if (dbias) {
    dim3 g(ceil_div(co, 32), (unsigned)std::min<long>(128, std::max<long>(1, npix / 256)));
    chan_reduce_kernel<2><<<g, 256, 0, s>>>(dy, dy, nullptr, nullptr, nullptr, 0, dbias, npix, co);
    MYOLO_LAUNCH_CHECK();
  }
  return 0;
}


// ------------------------------------------------------------------------------------------------
// generic conv backward for tiny maps and fp32 tensors (PPM bins, FFM attention FCs): reads the fp32 master weights directly
// ------------------------------------------------------------------------------------------------
__global__ void conv_small_dgrad_kernel(TensorView dy, TensorView dx, const float* __restrict__ w, int co, int ci, int k, int stride, int dil) {
  const long total = (long)dx.B * dx.H * dx.W * ci;
  const int pad = dil * (k / 2), taps = k * k;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ci);
    long p = i / ci;
    const int x = (int)(p % dx.W); p /= dx.W;
    const int y = (int)(p % dx.H);
    const int b = (int)(p / dx.H);
    float acc = 0.f;
    for (int ky = 0; ky < k; ++ky) {
      const int ny = y + pad - ky * dil;
      if (ny < 0 || ny % stride) continue;
      const int oy = ny / stride;
      if (oy >= dy.H) continue;
      for (int kx = 0; kx < k; ++kx) {
        const int nx = x + pad - kx * dil;
        if (nx < 0 || nx % stride) continue;
        const int ox = nx / stride;
        if (ox >= dy.W) continue;
        for (int o = 0; o < co; ++o) acc += ldv(dy, b, oy, ox, o) * w[((size_t)o * ci + c) * taps + ky * k + kx];
      }
    }
    stv(dx, b, y, x, c, ldv(dx, b, y, x, c) + acc);
  }
}
__global__ void conv_small_wgrad_kernel(TensorView x, TensorView dy, float* dW, int co, int ci, int k, int stride, int dil) {
  const int taps = k * k, pad = dil * (k / 2);
  const long total = (long)co * ci * taps;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int t = (int)(i % taps);
    const int c = (int)((i / taps) % ci);
    const int o = (int)(i / ((long)taps * ci));
    const int ky = t / k, kx = t % k;
    float acc = 0.f;
    for (int b = 0; b < dy.B; ++b)
      for (int oy = 0; oy < dy.H; ++oy) {
        const int iy = oy * stride - pad + ky * dil;
        if (iy < 0 || iy >= x.H) continue;
        for (int ox = 0; ox < dy.W; ++ox) {
          const int ix = ox * stride - pad + kx * dil;
          if (ix < 0 || ix >= x.W) continue;
          acc += ldv(dy, b, oy, ox, o) * ldv(x, b, iy, ix, c);
        }
      }
    atomicAdd(dW + i, acc);
  }
}
int launch_conv_small_bwd(const TensorView& x, const TensorView& dy, const TensorView* dx, const float* w, float* dW, float* dbias, int co,
                          int ci, int k, int stride, int dil, cudaStream_t s) {
  if (dx) {
    conv_small_dgrad_kernel<<<grid_for_t((long)dx->B * dx->H * dx->W * ci, 128), 128, 0, s>>>(dy, *dx, w, co, ci, k, stride, dil);
    MYOLO_LAUNCH_CHECK();
  }
  conv_small_wgrad_kernel<<<grid_for_t((long)co * ci * k * k, 128), 128, 0, s>>>(x, dy, dW, co, ci, k, stride, dil);
  MYOLO_LAUNCH_CHECK();
  if (dbias) {
    const long npix = (long)dy.B * dy.H * dy.W;
    dim3 g(ceil_div(co, 32), 1);
    chan_reduce_kernel<2><<<g, 256, 0, s>>>(dy, dy, nullptr, nullptr, nullptr, 0, dbias, npix, co);
    MYOLO_LAUNCH_CHECK();
  }
  return 0;
}

int launch_bias_grad(const TensorView& dy, float* dbias, int co, cudaStream_t s) {
  const long npix = (long)dy.B * dy.H * dy.W;
  dim3 g(ceil_div(co, 32), (unsigned)std::min<long>(128, std::max<long>(1, npix / 256)));
  chan_reduce_kernel<2><<<g, 256, 0, s>>>(dy, dy, nullptr, nullptr, nullptr, 0, dbias, npix, co);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// optimiser step over the FLAT parameter / gradient buffers (one launch for all 229 tensors; HBM-bound: 5 floats + 1 byte per element)
//   torch.optim.SGD(momentum, nesterov=True) with per-group lr / weight decay (reference train.py:108-126: pg0 BN weights, pg1 conv
//   weights with decay, pg2 biases), gradients unscaled by *inv_scale (loss scale x world size) and the step skipped when a non-finite
//   gradient was found (amp.GradScaler.step semantics, train.py:396-397); gradients are zeroed in the same pass (optimizer.zero_grad)
// ------------------------------------------------------------------------------------------------
__global__ void grads_check_finite_kernel(const float* __restrict__ g, long n, int* found_inf) {
  int bad = 0;
  const long n4 = n / 4;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(g)[i];
    bad |= !isfinite(v.x) | !isfinite(v.y) | !isfinite(v.z) | !isfinite(v.w);
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) bad |= !isfinite(g[n4 * 4 + threadIdx.x]);
  bad = __syncthreads_or(bad);
  if (threadIdx.x == 0 && bad) atomicOr(found_inf, 1);
}

struct SgdGroups { float lr[4]; float wd[4]; };
__global__ void sgd_step_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ buf, const unsigned char* __restrict__ group,
                                long n, SgdGroups gr, float momentum, int nesterov, const float* inv_scale, const int* found_inf, int zero_grad) {
  const bool skip = found_inf && *found_inf;
  const float is = inv_scale ? *inv_scale : 1.0f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    if (!skip) {
      const int k = group[i] & 3;
      const float w = p[i];
      float d = g[i] * is + gr.wd[k] * w;
      const float m = momentum * buf[i] + d;
      buf[i] = m;
      d = nesterov ? d + momentum * m : m;
      p[i] = w - gr.lr[k] * d;
    }
    if (zero_grad) g[i] = 0.f;
  }
}

// ------------------------------------------------------------------------------------------------
// torch.optim.Adam (reference train.py:128-129, --adam) behind amp.GradScaler, over the same flat buffers: 32 B of HBM traffic per
// element (p, g, exp_avg, exp_avg_sq read and written) + 1 B of group.  Bit-identical with GradScaler.unscale_ + torch's default
// CUDA implementation (_multi_tensor_adam, capturable=False), which runs one foreach kernel per line below, each rounding to fp32:
//   g  = g * inv_scale                               _amp_foreach_non_finite_check_and_unscale_
//   g  = fma(wd, p, g)          (wd != 0 only)       _foreach_add(g, p, alpha=wd)
//   m  = fma(1-b1, g - m, m)                         _foreach_lerp_(m, g, 1-b1), at::native::lerp for a weight < 0.5
//      (g - (g - m) * (1 - (1-b1)) for a weight >= 0.5)
//   v  = v * b2;  v = fma(1-b2, g*g, v)              _foreach_mul_, _foreach_addcmul_(v, g, g, 1-b2)
//   d  = sqrt(v) / bc2_sqrt + eps                    _foreach_sqrt, _foreach_div_(scalar list), _foreach_add_
//   p  = fma(-lr/bc1, m / d, p)                      _foreach_addcdiv_(p, m, d, scalar list)
// The explicit _rn intrinsics pin both the roundings and the contractions nvcc makes in torch's kernels.  The bias corrections are
// Python double arithmetic in torch (1 - beta**step, (lr / bc1) * -1, bc2 ** 0.5), rounded to fp32 when the scalar lists reach the
// kernels; they are computed here in double from the device step counter, so a skipped step (decided on the device) needs no host sync.
// ------------------------------------------------------------------------------------------------
struct AdamGroups { double lr[4]; float wd[4]; };
struct AdamScalars { float step_size, bc2_sqrt; };

// step k = 1, 2, ...: what torch hands its kernels for group lr (CUDA's double sqrt and division are correctly rounded, as glibc's are;
// tests/test_gpu_optim.py compares the double bias corrections with Python's for every k up to 10^6).
// beta^k rounded to double: CUDA's pow (2 ulp) differs from glibc's for some k (e.g. 0.937^3), so the power is taken by squaring in
// double-double arithmetic (error ~ 2 log2(k) * 2^-104), which rounds to the correctly rounded double that glibc's pow returns
__device__ __forceinline__ void dd_mul(double& hi, double& lo, double bh, double bl) {
  const double p = hi * bh;
  double e = fma(hi, bh, -p);
  e = fma(hi, bl, fma(lo, bh, e));
  hi = p + e;
  lo = e - (hi - p);
}
__device__ __forceinline__ double bias_correction(double beta, int k) {
  double rh = 1.0, rl = 0.0, xh = beta, xl = 0.0;
  for (unsigned e = (unsigned)k; e; e >>= 1) {
    if (e & 1) dd_mul(rh, rl, xh, xl);
    if (e > 1) dd_mul(xh, xl, xh, xl);
  }
  return 1.0 - (rh + rl);
}
__device__ __forceinline__ AdamScalars adam_scalars(int k, double lr, double beta1, double beta2) {
  return AdamScalars{(float)((lr / bias_correction(beta1, k)) * -1.0), (float)sqrt(bias_correction(beta2, k))};
}

__device__ __forceinline__ void adam_element(float& p, float& g, float& m, float& v, float is, float wd, float w1, float b2, float w2,
                                             float eps, AdamScalars sc) {
  float gr = __fmul_rn(g, is);
  if (wd != 0.f) gr = __fmaf_rn(wd, p, gr);
  const float diff = __fsub_rn(gr, m);
  m = fabsf(w1) < 0.5f ? __fmaf_rn(w1, diff, m) : __fmaf_rn(-diff, __fsub_rn(1.f, w1), gr);
  v = __fmaf_rn(w2, __fmul_rn(gr, gr), __fmul_rn(v, b2));
  const float d = __fadd_rn(__fdiv_rn(__fsqrt_rn(v), sc.bc2_sqrt), eps);
  p = __fmaf_rn(sc.step_size, __fdiv_rn(m, d), p);
}

__global__ void adam_step_kernel(float* __restrict__ p, float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                                 const unsigned char* __restrict__ group, long n, AdamGroups gr, int n_groups, double beta1, double beta2,
                                 float w1, float b2, float w2, float eps, const int* steps, const float* inv_scale, const int* found_inf,
                                 int zero_grad) {
  __shared__ AdamScalars sc[4];
  __shared__ float swd[4];
  const bool skip = found_inf && *found_inf;
  const float is = inv_scale ? *inv_scale : 1.0f;
  if (threadIdx.x < n_groups) {
    double lr = gr.lr[0];
    float wd = gr.wd[0];
#pragma unroll
    for (int j = 1; j < 4; ++j)                       // constant indices: the kernel parameters stay out of local memory
      if (threadIdx.x == j) { lr = gr.lr[j]; wd = gr.wd[j]; }
    swd[threadIdx.x] = wd;
    if (!skip) sc[threadIdx.x] = adam_scalars(*steps + 1, lr, beta1, beta2);
  }
  __syncthreads();
  const long n4 = n / 4;
  const long stride = (long)gridDim.x * blockDim.x;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 gv = reinterpret_cast<float4*>(g)[i];
    if (!skip) {
      float4 pv = reinterpret_cast<float4*>(p)[i], mv = reinterpret_cast<float4*>(m)[i], vv = reinterpret_cast<float4*>(v)[i];
      const uchar4 k = reinterpret_cast<const uchar4*>(group)[i];
      adam_element(pv.x, gv.x, mv.x, vv.x, is, swd[k.x & 3], w1, b2, w2, eps, sc[k.x & 3]);
      adam_element(pv.y, gv.y, mv.y, vv.y, is, swd[k.y & 3], w1, b2, w2, eps, sc[k.y & 3]);
      adam_element(pv.z, gv.z, mv.z, vv.z, is, swd[k.z & 3], w1, b2, w2, eps, sc[k.z & 3]);
      adam_element(pv.w, gv.w, mv.w, vv.w, is, swd[k.w & 3], w1, b2, w2, eps, sc[k.w & 3]);
      reinterpret_cast<float4*>(p)[i] = pv;
      reinterpret_cast<float4*>(m)[i] = mv;
      reinterpret_cast<float4*>(v)[i] = vv;
    }
    if (zero_grad) reinterpret_cast<float4*>(g)[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  const long i = n4 * 4 + blockIdx.x * (long)blockDim.x + threadIdx.x;     // the tail of n % 4 elements
  if (i < n) {
    if (!skip) {
      const int k = group[i] & 3;
      adam_element(p[i], g[i], m[i], v[i], is, swd[k], w1, b2, w2, eps, sc[k]);
    }
    if (zero_grad) g[i] = 0.f;
  }
}

__global__ void adam_scalars_kernel(const int* steps, long n, double lr, double beta1, double beta2, float* step_size, float* bc2_sqrt,
                                    double* bc1, double* bc2) {
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    const AdamScalars sc = adam_scalars(steps[i], lr, beta1, beta2);
    step_size[i] = sc.step_size;
    bc2_sqrt[i] = sc.bc2_sqrt;
    bc1[i] = bias_correction(beta1, steps[i]);
    bc2[i] = bias_correction(beta2, steps[i]);
  }
}

// ------------------------------------------------------------------------------------------------
// ModelEMA.update (reference utils/torch_utils.py:290-300) over every floating-point state_dict entry: one CTA per chunk of the device
// table, 12 B of HBM traffic per fp32 element (8 B for an fp16 EMA).  The reference runs three torch ops per entry, each rounding to its
// own dtype; the _rn intrinsics keep nvcc from contracting them into an FMA:
//   v *= d                   rn(v * df)                   fp16 EMA: half_rn(float(v) * df)      (opmath float, stored as half)
//   t  = (1. - d) * msd[k]   rn(d1f * m)                  fp32 (the source is the fp32 training model)
//   v += t                   rn(v + t)                    fp16 EMA: half_rn(float(v) + t)       (promoted to fp32, stored as half)
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float ema_f32(float v, float m, float df, float d1f) {
  return __fadd_rn(__fmul_rn(v, df), __fmul_rn(d1f, m));
}
__device__ __forceinline__ __half ema_f16(__half v, float m, float df, float d1f) {
  const float a = __half2float(__float2half_rn(__fmul_rn(__half2float(v), df)));
  return __float2half_rn(__fadd_rn(a, __fmul_rn(d1f, m)));
}

__global__ void __launch_bounds__(256) ema_update_kernel(const myolo_ema_chunk* __restrict__ chunks, float df, float d1f) {
  const myolo_ema_chunk c = chunks[blockIdx.x];
  const float* __restrict__ src = c.src;
  const int n = c.n;
  int i0 = 0;                                              // first element of the scalar part
  if (c.dtype == MYOLO_F32) {
    float* __restrict__ v = static_cast<float*>(c.ema);
    if (((reinterpret_cast<uintptr_t>(v) | reinterpret_cast<uintptr_t>(src)) & 15) == 0) {
      const int n4 = n >> 2;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        float4 a = reinterpret_cast<float4*>(v)[i];
        const float4 m = __ldg(reinterpret_cast<const float4*>(src) + i);
        a.x = ema_f32(a.x, m.x, df, d1f);
        a.y = ema_f32(a.y, m.y, df, d1f);
        a.z = ema_f32(a.z, m.z, df, d1f);
        a.w = ema_f32(a.w, m.w, df, d1f);
        reinterpret_cast<float4*>(v)[i] = a;
      }
      i0 = n4 * 4;
    }
    for (int i = i0 + threadIdx.x; i < n; i += blockDim.x) v[i] = ema_f32(v[i], __ldg(src + i), df, d1f);
  } else {
    __half* __restrict__ v = static_cast<__half*>(c.ema);
    if ((reinterpret_cast<uintptr_t>(v) & 7) == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
      const int n4 = n >> 2;
      for (int i = threadIdx.x; i < n4; i += blockDim.x) {
        uint2 raw = reinterpret_cast<uint2*>(v)[i];
        __half2* h = reinterpret_cast<__half2*>(&raw);
        const float4 m = __ldg(reinterpret_cast<const float4*>(src) + i);
        h[0] = __halves2half2(ema_f16(__low2half(h[0]), m.x, df, d1f), ema_f16(__high2half(h[0]), m.y, df, d1f));
        h[1] = __halves2half2(ema_f16(__low2half(h[1]), m.z, df, d1f), ema_f16(__high2half(h[1]), m.w, df, d1f));
        reinterpret_cast<uint2*>(v)[i] = raw;
      }
      i0 = n4 * 4;
    }
    for (int i = i0 + threadIdx.x; i < n; i += blockDim.x) v[i] = ema_f16(v[i], __ldg(src + i), df, d1f);
  }
}

}  // namespace myolo

using namespace myolo;

extern "C" int64_t myolo_seg_focal_loss_workspace_bytes(void) { return (int64_t)kSegWfHead; }

extern "C" int myolo_seg_focal_loss(const float* x, const int64_t* labels, int B, int C, int H, int W, int ignore_index, const float* weights,
                                    float gamma, int reduction, float* loss_out, void* ws, int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_seg_focal_loss");
  MYOLO_REQUIRE(x && labels && loss_out && ws && B > 0 && C > 0 && H > 0 && W > 0, "seg_focal_loss: bad arguments");
  MYOLO_REQUIRE(reduction == MYOLO_REDUCTION_MEAN || reduction == MYOLO_REDUCTION_SUM, "seg_focal_loss: reduction must be mean or sum");
  MYOLO_REQUIRE(workspace_bytes >= myolo_seg_focal_loss_workspace_bytes(), "seg_focal_loss: workspace too small");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(gamma >= 0.f && isfinite(gamma), "seg_focal_loss: gamma must be finite and >= 0, got %g", (double)gamma);
  const long n = (long)B * H * W;
  SegWfSt* st = reinterpret_cast<SegWfSt*>(ws);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(ws, 0, sizeof(SegWfSt), s));
  seg_focal_nchw_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(x, reinterpret_cast<const long long*>(labels), B, C, (long)H * W, ignore_index, weights,
                                                             gamma, st);
  MYOLO_LAUNCH_CHECK();
  seg_wf_finalize_kernel<<<1, 1, 0, s>>>(st, gamma, (float)n, reduction == MYOLO_REDUCTION_SUM, loss_out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_seg_focal_loss_backward(const float* x, const int64_t* labels, int B, int C, int H, int W, int ignore_index,
                                             const float* weights, float gamma, const float* grad_out, float* dx, const void* ws,
                                             int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_seg_focal_loss_backward");
  MYOLO_REQUIRE(x && labels && grad_out && dx && ws && B > 0 && C > 0 && H > 0 && W > 0, "seg_focal_loss_backward: bad arguments");
  MYOLO_REQUIRE(workspace_bytes >= myolo_seg_focal_loss_workspace_bytes(), "seg_focal_loss_backward: workspace too small");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(gamma >= 0.f && isfinite(gamma), "seg_focal_loss_backward: gamma must be finite and >= 0, got %g", (double)gamma);
  const long n = (long)B * H * W;
  seg_focal_nchw_bwd_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(x, reinterpret_cast<const long long*>(labels), B, C, (long)H * W, ignore_index,
                                                                 weights, gamma, reinterpret_cast<const SegWfSt*>(ws), grad_out, dx);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int64_t myolo_seg_ohem_loss_workspace_bytes(int B, int H, int W) { return (int64_t)ohem_scratch_bytes((long)B * H * W); }

extern "C" int myolo_seg_ohem_loss(const float* x, const int64_t* labels, int B, int C, int H, int W, int ignore_index, float thresh_t,
                                   float* loss_out, void* ws, int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_seg_ohem_loss");
  MYOLO_REQUIRE(x && labels && loss_out && ws && B > 0 && C > 0 && H > 0 && W > 0, "seg_ohem_loss: bad arguments");
  MYOLO_REQUIRE(workspace_bytes >= myolo_seg_ohem_loss_workspace_bytes(B, H, W), "seg_ohem_loss: workspace too small");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  const long n = (long)B * H * W;
  OhemScratch oh = ohem_scratch(ws, n);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(ws, 0, oh.head, s));
  count_valid_kernel<<<grid_for_t(n, 256, 132 * 8), 256, 0, s>>>(reinterpret_cast<const long long*>(labels), n, ignore_index, C,
                                                                  &oh.st->n_valid);
  MYOLO_LAUNCH_CHECK();
  ohem_ce_nchw_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(x, reinterpret_cast<const long long*>(labels), B, C, (long)H * W, ignore_index,
                                                          oh.loss);
  MYOLO_LAUNCH_CHECK();
  if (int rc = ohem_select(oh.loss, n, &oh.st->n_valid, thresh_t, oh.st, oh.ties, s)) return rc;
  ohem_finalize_kernel<<<1, 1, 0, s>>>(oh.st, loss_out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_seg_ohem_loss_backward(const float* x, const int64_t* labels, int B, int C, int H, int W, int ignore_index,
                                            const float* grad_out, float* dx, const void* ws, int64_t workspace_bytes, void* stream) {
  NvtxRange nvtx_("myolo_seg_ohem_loss_backward");
  MYOLO_REQUIRE(x && labels && grad_out && dx && ws && B > 0 && C > 0 && H > 0 && W > 0, "seg_ohem_loss_backward: bad arguments");
  MYOLO_REQUIRE(workspace_bytes >= myolo_seg_ohem_loss_workspace_bytes(B, H, W), "seg_ohem_loss_backward: workspace too small");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  const long n = (long)B * H * W;
  OhemScratch oh = ohem_scratch(const_cast<void*>(ws), n);
  ohem_ce_nchw_bwd_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(x, reinterpret_cast<const long long*>(labels), B, C, (long)H * W, ignore_index,
                                                              oh.loss, oh.st, grad_out, dx);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_grads_check_finite(const float* g, int64_t n, int32_t* found_inf, void* stream) {
  MYOLO_REQUIRE(g && found_inf && n > 0, "grads_check_finite: bad arguments");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "grads_check_finite: gradient buffer must be 16-byte aligned");
  MYOLO_CHECK_CUDA(cudaMemsetAsync(found_inf, 0, sizeof(int), s));
  grads_check_finite_kernel<<<grid_for_t(std::max<long>(1, n / 4), 256, 132 * 8), 256, 0, s>>>(g, n, found_inf);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_sgd_step(float* p, float* g, float* buf, const uint8_t* group, int64_t n, const float* lr, const float* wd, int n_groups,
                              float momentum, int nesterov, const float* inv_scale, const int32_t* found_inf, int zero_grad, void* stream) {
  NvtxRange nvtx_("myolo_sgd_step");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(p && g && buf && group && n > 0 && n_groups >= 1 && n_groups <= 4, "sgd_step: bad arguments");
  SgdGroups gr{};
  for (int i = 0; i < n_groups; ++i) { gr.lr[i] = lr[i]; gr.wd[i] = wd[i]; }
  sgd_step_kernel<<<grid_for_t(n, 256, 132 * 8), 256, 0, s>>>(p, g, buf, group, n, gr, momentum, nesterov, inv_scale, found_inf, zero_grad);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_adam_step(float* p, float* g, float* m, float* v, const uint8_t* group, int64_t n, const double* lr, const float* wd,
                               int n_groups, double beta1, double beta2, double eps, const int32_t* steps, const float* inv_scale,
                               const int32_t* found_inf, int zero_grad, void* stream) {
  NvtxRange nvtx_("myolo_adam_step");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(p && g && m && v && group && steps && n > 0 && n_groups >= 1 && n_groups <= 4, "adam_step: bad arguments");
  MYOLO_REQUIRE(((reinterpret_cast<uintptr_t>(p) | reinterpret_cast<uintptr_t>(g) | reinterpret_cast<uintptr_t>(m) |
                  reinterpret_cast<uintptr_t>(v)) & 15) == 0 && (reinterpret_cast<uintptr_t>(group) & 3) == 0,
                "adam_step: buffers must be 16-byte aligned (group: 4-byte)");
  AdamGroups gr{};
  for (int i = 0; i < n_groups; ++i) { gr.lr[i] = lr[i]; gr.wd[i] = wd[i]; }
  // torch's scalars: 1 - beta1 (lerp weight), beta2, 1 - beta2 and eps, each Python double rounded to fp32
  adam_step_kernel<<<grid_for_t(std::max<long>(1, n / 4), 256, 132 * 8), 256, 0, s>>>(
      p, g, m, v, group, n, gr, n_groups, beta1, beta2, (float)(1.0 - beta1), (float)beta2, (float)(1.0 - beta2), (float)eps, steps,
      inv_scale, found_inf, zero_grad);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_adam_scalars(const int32_t* steps, int64_t n, double lr, double beta1, double beta2, float* step_size, float* bc2_sqrt,
                                  double* bc1, double* bc2, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(steps && step_size && bc2_sqrt && bc1 && bc2 && n > 0, "adam_scalars: bad arguments");
  adam_scalars_kernel<<<grid_for_t(n, 256), 256, 0, s>>>(steps, n, lr, beta1, beta2, step_size, bc2_sqrt, bc1, bc2);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_ema_update(const myolo_ema_chunk* chunks, int n_chunks, double decay, void* stream) {
  NvtxRange nvtx_("myolo_ema_update");
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(chunks && n_chunks > 0, "ema_update: empty chunk table");
  MYOLO_REQUIRE(decay >= 0.0 && decay <= 1.0, "ema_update: decay %g outside [0, 1]", decay);
  MYOLO_REQUIRE((reinterpret_cast<uintptr_t>(chunks) & 7) == 0, "ema_update: chunk table must be 8-byte aligned");
  // torch hands `d` and `1. - d` (Python doubles) to fp32-math kernels: each is rounded to fp32 once
  ema_update_kernel<<<n_chunks, 256, 0, s>>>(chunks, (float)decay, (float)(1.0 - decay));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
