// Training-mode kernels (see train.h).  Correct-first implementations: the data gradients of all convolutions reuse the wgmma
// implicit-GEMM kernel (a conv of dY with flipped/transposed weights); weight gradients run on legacy mma.sync with split-K
// atomics; everything else is plain coalesced CUDA.  Reference semantics: torch.autograd through models/common.py / models/yolo.py
// in train mode (BatchNorm with batch statistics, eps 1e-3, momentum 0.03: reference utils/torch_utils.py:150-152).
#include <algorithm>

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
    for (long p = p0 + lane_p; p < p1; p += 8) {
      const size_t off = (size_t)p * a.ctot + c;
      if (MODE == 0) {
        const float u = __half2float(reinterpret_cast<const __half*>(a.base)[off]);
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
template <int MODE>
__global__ void __launch_bounds__(256) chan_reduce_v_kernel(TensorView a, TensorView bview, const float* __restrict__ stats,
                                                            const float* __restrict__ gamma, const float* __restrict__ beta, int act,
                                                            float* out, long npix, int C, BnParams bn, float* stats_out,
                                                            unsigned* ticket, float* final_out) {
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
    for (long p = (long)blockIdx.x * lanes + lane; p < npix; p += (long)gridDim.x * lanes) {
      const uint4 q = *reinterpret_cast<const uint4*>(ab + (size_t)p * a.ctot + cv * 8);
      const __half* h = reinterpret_cast<const __half*>(&q);
      if (MODE == 0) {
#pragma unroll
        for (int k = 0; k < 8; ++k) { const float u = __half2float(h[k]); s0[k] += u; s1[k] += u * u; }
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
  for (int c = t; c < C; c += 256) {
    const float x0 = __ldcg(out + c), x1 = __ldcg(out + C + c);
    out[c] = 0.f;
    out[C + c] = 0.f;
    if (final_out) { final_out[c] = x0; final_out[C + c] = x1; }
    if (MODE == 0) {
      const float n = (float)npix;
      const float mean = x0 / n;
      const float var = fmaxf(x1 / n - mean * mean, 0.f);          // biased variance normalises (F.batch_norm, training=True)
      stats_out[c] = mean;
      stats_out[C + c] = rsqrtf(var + bn.eps);
      if (bn.running_mean) {                                       // running stats: unbiased variance, momentum 0.03
        bn.running_mean[c] = (1.f - bn.momentum) * bn.running_mean[c] + bn.momentum * mean;
        bn.running_var[c] = (1.f - bn.momentum) * bn.running_var[c] + bn.momentum * var * (n / fmaxf(n - 1.f, 1.f));
      }
    } else {
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

__global__ void bn_finalize_kernel(float* sums, float* stats, BnParams bn, long npix) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= bn.C) return;
  const float n = (float)npix;
  const float mean = sums[c] / n;
  const float var = fmaxf(sums[bn.C + c] / n - mean * mean, 0.f);           // biased variance normalises (F.batch_norm, training=True)
  stats[c] = mean;
  stats[bn.C + c] = rsqrtf(var + bn.eps);
  if (bn.running_mean) {                                                       // running stats: unbiased variance, momentum 0.03
    bn.running_mean[c] = (1.f - bn.momentum) * bn.running_mean[c] + bn.momentum * mean;
    bn.running_var[c] = (1.f - bn.momentum) * bn.running_var[c] + bn.momentum * var * (n / fmaxf(n - 1.f, 1.f));
  }
}

// deferred running statistics: one launch applies r <- (1-m) r + m * stat for every BN layer of a plan from the sums its last forward left
__global__ void __launch_bounds__(256) bn_apply_running_kernel(const RunningJob* __restrict__ jobs) {
  const RunningJob j = jobs[blockIdx.x];
  const float n = (float)j.npix;
  for (int c = threadIdx.x; c < j.C; c += 256) {
    const float mean = j.sums[c] / n;
    const float var = fmaxf(j.sums[j.C + c] / n - mean * mean, 0.f);
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
  // scratch (zero on entry, left zero by the kernel): 2*C sums, 2*C final sums (backward), the completion ticket
  if (u.C % 8 == 0 && u.C <= 2048 && u.ctot % 8 == 0) {
    MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<0>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, u, (const float*)nullptr,
                                (const float*)nullptr, (const float*)nullptr, 0, scratch, npix, u.C, bn, stats,
                                reinterpret_cast<unsigned*>(scratch + 4 * u.C), defer_running ? scratch + 2 * u.C : (float*)nullptr));
    g_launch_count++;
    return 0;
  }
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));
  dim3 g(ceil_div(u.C, 32), (unsigned)std::min<long>(256, std::max<long>(1, npix / 256)));
  chan_reduce_kernel<0><<<g, 256, 0, s>>>(u, u, nullptr, nullptr, nullptr, 0, scratch, npix, u.C);
  MYOLO_LAUNCH_CHECK();
  bn_finalize_kernel<<<ceil_div(u.C, 128), 128, 0, s>>>(scratch, stats, bn, npix);
  MYOLO_LAUNCH_CHECK();
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch, 0, (2 * (size_t)u.C) * sizeof(float), s));    // contract of the scratch: zero between launches
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
                                  float inv_n) {
  pdl_enter();
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
int launch_bn_act_bwd(const TensorView& u, const TensorView& dy, const TensorView& du, const TensorView* d_res, const BnParams& bn,
                      const float* stats, int act, float* scratch, cudaStream_t s) {
  MYOLO_REQUIRE(u.C % 8 == 0 && dy.C == u.C && du.C == u.C && dy.ctot % 8 == 0 && du.ctot % 8 == 0 && u.ctot % 8 == 0, "bn_act_bwd: bad views");
  MYOLO_REQUIRE(!d_res || (d_res->C == u.C && d_res->ctot % 8 == 0), "bn_act_bwd: bad residual gradient view");
  const long npix = (long)u.B * u.H * u.W;
  const float* sums = scratch;
  if (u.C <= 2048) {
    MYOLO_CHECK_CUDA(launch_pdl(chan_reduce_v_kernel<1>, dim3(reduce_v_grid(npix, u.C)), dim3(256), 0, s, u, dy, stats, (const float*)bn.gamma,
                                (const float*)bn.beta, act, scratch, npix, u.C, bn, (float*)nullptr,
                                reinterpret_cast<unsigned*>(scratch + 4 * u.C), scratch + 2 * u.C));
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
                              d_res != nullptr, (const float*)bn.gamma, (const float*)bn.beta, stats, sums, act, 1.0f / (float)npix));
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

// pass 1: one thread per FULL-resolution pixel: interpolated logits from the 4 low-res neighbours -> softmax -> (p - onehot) written as
// NC_PAD fp32 per pixel (zeros for ignored pixels); the pixel's loss is reduced per warp.
template <int NC, int NC_PAD>
__global__ void seg_ce_pixel_kernel(TensorView lo, const long long* __restrict__ labels, int H, int W, int ignore_index, float* __restrict__ g,
                                    float* loss_sum) {
  const long total = (long)lo.B * H * W;
  float loss_local = 0.f;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int X = (int)(i % W);
    const int Y = (int)((i / W) % H);
    const int b = (int)(i / ((long)W * H));
    const long long t = labels[i];
    float v[NC_PAD];
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
      loss_local += __logf(ssum) + m - zt;
    }
    float4* dst = reinterpret_cast<float4*>(g + (size_t)i * NC_PAD);
#pragma unroll
    for (int c = 0; c < NC_PAD; c += 4) dst[c / 4] = make_float4(v[c], v[c + 1], v[c + 2], v[c + 3]);
  }
  loss_local = warp_sum(loss_local);
  if ((threadIdx.x & 31) == 0 && loss_local != 0.f) atomicAdd(loss_sum, loss_local);
}

// pass 2: adjoint of the bilinear upsample, gathered per low-res pixel (x a chunk of its footprint rows) from the per-pixel gradients
template <int NC, int NC_PAD>
__global__ void seg_ce_gather_kernel(const float* __restrict__ g, int H, int W, TensorView dlo, float factor, const float* __restrict__ scale_dev,
                                     const unsigned long long* __restrict__ n_valid, int rsplit) {
  const long total = (long)dlo.B * dlo.H * dlo.W * rsplit;
  const unsigned long long nv = *n_valid;
  const float coef = nv ? factor * (scale_dev ? *scale_dev : 1.0f) / (float)nv : 0.f;
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
        const float wgt = wy * ((b0 == x ? v0 : 0.f) + (b1 == x ? v1 : 0.f));
        if (wgt == 0.f) continue;
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
int launch_seg_ce_fused(const TensorView& lo, int n_cls, const long long* labels, int H, int W, int ignore_index, const TensorView& dlo,
                        float factor, const float* scale_dev, void* scratch16, float* gbuf, float* loss_out, cudaStream_t s) {
  MYOLO_REQUIRE(lo.dtype == MYOLO_F32 && dlo.dtype == MYOLO_F32 && n_cls >= 1 && n_cls <= 32 && lo.C >= n_cls && labels && scratch16 && gbuf,
                "seg_ce_fused: fp32 low-resolution logits with <= 32 classes expected");
  unsigned long long* n_valid = reinterpret_cast<unsigned long long*>(scratch16);
  float* loss_sum = reinterpret_cast<float*>(n_valid + 1);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(scratch16, 0, 16, s));
  const long n = (long)lo.B * H * W;
  count_valid_kernel<<<grid_for_t(n, 256, 132 * 8), 256, 0, s>>>(labels, n, ignore_index, n_cls, n_valid);
  MYOLO_LAUNCH_CHECK();
  const int rsplit = 4;
  const int g1 = grid_for_t(n, 128), g2 = grid_for_t((long)lo.B * lo.H * lo.W * rsplit, 128);
  if (n_cls == 19) {
    seg_ce_pixel_kernel<19, 20><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, loss_sum);
    MYOLO_LAUNCH_CHECK();
    seg_ce_gather_kernel<19, 20><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, n_valid, rsplit);
  } else if (n_cls <= 20) {
    MYOLO_REQUIRE(false, "seg_ce_fused: instantiate the kernels for %d classes (19 and 21..32 are built)", n_cls);
  } else {
    MYOLO_REQUIRE(n_cls == 32, "seg_ce_fused: instantiate the kernels for %d classes (19 and 32 are built)", n_cls);
    seg_ce_pixel_kernel<32, 32><<<g1, 128, 0, s>>>(lo, labels, H, W, ignore_index, gbuf, loss_sum);
    MYOLO_LAUNCH_CHECK();
    seg_ce_gather_kernel<32, 32><<<g2, 128, 0, s>>>(gbuf, H, W, dlo, factor, scale_dev, n_valid, rsplit);
  }
  MYOLO_LAUNCH_CHECK();
  seg_ce_finalize_kernel<<<1, 1, 0, s>>>(loss_sum, n_valid, loss_out);
  MYOLO_LAUNCH_CHECK();
  return 0;
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
int launch_grads_check_finite(const float* g, long n, int* found_inf, cudaStream_t s) {
  MYOLO_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "grads_check_finite: gradient buffer must be 16-byte aligned");
  MYOLO_CHECK_CUDA(cudaMemsetAsync(found_inf, 0, sizeof(int), s));
  grads_check_finite_kernel<<<grid_for_t(std::max<long>(1, n / 4), 256, 132 * 8), 256, 0, s>>>(g, n, found_inf);
  MYOLO_LAUNCH_CHECK();
  return 0;
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
int launch_sgd_step(float* p, float* g, float* buf, const unsigned char* group, long n, const float* lr, const float* wd, int n_groups,
                    float momentum, int nesterov, const float* inv_scale, const int* found_inf, int zero_grad, cudaStream_t s) {
  MYOLO_REQUIRE(p && g && buf && group && n > 0 && n_groups >= 1 && n_groups <= 4, "sgd_step: bad arguments");
  SgdGroups gr{};
  for (int i = 0; i < n_groups; ++i) { gr.lr[i] = lr[i]; gr.wd[i] = wd[i]; }
  sgd_step_kernel<<<grid_for_t(n, 256, 132 * 8), 256, 0, s>>>(p, g, buf, group, n, gr, momentum, nesterov, inv_scale, found_inf, zero_grad);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo
