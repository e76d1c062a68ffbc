// Generic CUDA-core conv (+bias+act+residual) on NHWC views.  Used for shapes the wgmma kernel does not take
// (maps smaller than one 128-pixel tile: PPM 1x1..6x6 bins, FFM attention FCs, P5 at tiny test resolutions) and,
// with MYOLO_FORCE_SIMT=1, as an independent on-device cross-check of the tensor-core path.
// One warp computes one output pixel x 32 consecutive output channels; lanes split K (coalesced 16-byte loads of both
// the activation pixel and the weight row) and reduce with shuffles.
#include <algorithm>

#include "conv.h"

namespace myolo {

template <typename TIn>
__device__ __forceinline__ void load8(const TIn* p, float (&f)[8]);
template <>
__device__ __forceinline__ void load8<__half>(const __half* p, float (&f)[8]) {
  const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
template <>
__device__ __forceinline__ void load8<float>(const float* p, float (&f)[8]) {
  const float4 a = __ldg(reinterpret_cast<const float4*>(p));
  const float4 b = __ldg(reinterpret_cast<const float4*>(p) + 1);
  f[0] = a.x; f[1] = a.y; f[2] = a.z; f[3] = a.w;
  f[4] = b.x; f[5] = b.y; f[6] = b.z; f[7] = b.w;
}

struct SimtParams {
  const void* in; int in_ctot; int H, W, Ci;      // Ci = Ci_pad (multiple of 8)
  void* out; int out_ctot; int out_f32; int Ho, Wo, Co;
  const __half* res; int res_ctot;
  const __half* w; const float* bias;
  int k, stride, dil, act, B;
};

template <typename TIn>
__device__ __forceinline__ void conv_simt_body(const SimtParams& p) {
  const int lane = threadIdx.x & 31;
  const int warp_global = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int co_groups = (p.Co + 7) / 8;
  const long total = (long)p.B * p.Ho * p.Wo * co_groups;
  const int nwarps = (gridDim.x * blockDim.x) >> 5;
  const int taps = p.k * p.k;
  const int pad = p.dil * (p.k / 2);
  const int Kt = taps * p.Ci;
  for (long item = warp_global; item < total; item += nwarps) {
    const int cg = (int)(item % co_groups);
    const long pix = item / co_groups;
    const int ox = (int)(pix % p.Wo);
    const int oy = (int)((pix / p.Wo) % p.Ho);
    const int b = (int)(pix / ((long)p.Wo * p.Ho));
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    for (int t = 0; t < taps; ++t) {
      const int iy = oy * p.stride - pad + (t / p.k) * p.dil;
      const int ix = ox * p.stride - pad + (t % p.k) * p.dil;
      if (iy < 0 || iy >= p.H || ix < 0 || ix >= p.W) continue;
      const TIn* ip = reinterpret_cast<const TIn*>(p.in) + (((size_t)b * p.H + iy) * p.W + ix) * p.in_ctot;
      for (int c = lane * 8; c < p.Ci; c += 256) {
        float xv[8];
        load8<TIn>(ip + c, xv);
#pragma unroll
        for (int o = 0; o < 8; ++o) {
          const int co = cg * 8 + o;
          float wv[8];
          load8<__half>(p.w + (size_t)co * Kt + t * p.Ci + c, wv);
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[o] = fmaf(xv[i], wv[i], acc[o]);
        }
      }
    }
#pragma unroll
    for (int o = 0; o < 8; ++o) {
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) acc[o] += __shfl_xor_sync(0xffffffffu, acc[o], s);
    }
    if (lane < 8) {
      const int co = cg * 8 + lane;
      if (co < p.Co) {
        float v = 0.f;
#pragma unroll
        for (int o = 0; o < 8; ++o) v = (o == lane) ? acc[o] : v;
        v += p.bias[co];
        v = apply_act(v, p.act);
        const size_t opix = ((size_t)b * p.Ho + oy) * p.Wo + ox;
        if (p.res) v += __half2float(p.res[opix * p.res_ctot + co]);
        if (p.out_f32) reinterpret_cast<float*>(p.out)[opix * p.out_ctot + co] = v;
        else reinterpret_cast<__half*>(p.out)[opix * p.out_ctot + co] = __float2half_rn(v);
      }
    }
  }
}

template <typename TIn>
__global__ void __launch_bounds__(256) conv_simt_kernel(SimtParams p) {
  pdl_enter();
  conv_simt_body<TIn>(p);
}
// up to 4 small convolutions of the same input type in ONE launch (the 1x1 convs on the pooled bins of PyramidPooling): blockIdx.y = member
struct SimtGroup { SimtParams p[4]; };
template <typename TIn>
__global__ void __launch_bounds__(256) conv_simt_group_kernel(SimtGroup g) {
  pdl_enter();
  conv_simt_body<TIn>(g.p[blockIdx.y]);
}

static int fill_simt_params(const ConvOp& op, SimtParams& p) {
  p.in = op.in.base; p.in_ctot = op.in.ctot; p.H = op.in.H; p.W = op.in.W; p.Ci = op.Ci_pad;
  p.out = op.out.base; p.out_ctot = op.out.ctot; p.out_f32 = op.out.dtype == MYOLO_F32; p.Ho = op.out.H; p.Wo = op.out.W;
  p.Co = op.Co;
  p.res = op.has_res ? reinterpret_cast<const __half*>(op.res.base) : nullptr; p.res_ctot = op.has_res ? op.res.ctot : 0;
  p.w = op.w; p.bias = op.bias; p.k = op.k; p.stride = op.stride; p.dil = op.dil; p.act = op.act; p.B = op.in.B;
  MYOLO_REQUIRE(op.Ci_pad % 8 == 0 && op.in.ctot % (op.in.dtype == MYOLO_F16 ? 8 : 4) == 0, "conv_simt: Ci_pad %d / ctot %d alignment",
                op.Ci_pad, op.in.ctot);
  MYOLO_REQUIRE(op.in.C >= op.Ci_pad, "conv_simt: input view has %d channels, packed weights expect %d", op.in.C, op.Ci_pad);
  return 0;
}
int conv_simt_launch_group(const ConvOp* const* ops, int n, cudaStream_t stream) {
  MYOLO_REQUIRE(n >= 1 && n <= 4, "conv_simt_group: %d members", n);
  SimtGroup g;
  long most = 1;
  for (int i = 0; i < n; ++i) {
    MYOLO_REQUIRE(ops[i]->in.dtype == ops[0]->in.dtype, "conv_simt_group: mixed input types");
    int rc = fill_simt_params(*ops[i], g.p[i]);
    if (rc) return rc;
    most = std::max(most, ((long)g.p[i].B * g.p[i].Ho * g.p[i].Wo * ((g.p[i].Co + 7) / 8) + 7) / 8);
  }
  if (most > 132 * 16) most = 132 * 16;
  if (ops[0]->in.dtype == MYOLO_F16) MYOLO_CHECK_CUDA(launch_pdl(conv_simt_group_kernel<__half>, dim3((int)most, n), dim3(256), 0, stream, g));
  else MYOLO_CHECK_CUDA(launch_pdl(conv_simt_group_kernel<float>, dim3((int)most, n), dim3(256), 0, stream, g));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

int conv_simt_launch(const ConvOp& op, cudaStream_t stream) {
  SimtParams p;
  p.in = op.in.base; p.in_ctot = op.in.ctot; p.H = op.in.H; p.W = op.in.W; p.Ci = op.Ci_pad;
  p.out = op.out.base; p.out_ctot = op.out.ctot; p.out_f32 = op.out.dtype == MYOLO_F32; p.Ho = op.out.H; p.Wo = op.out.W;
  p.Co = op.Co;
  p.res = op.has_res ? reinterpret_cast<const __half*>(op.res.base) : nullptr; p.res_ctot = op.has_res ? op.res.ctot : 0;
  p.w = op.w; p.bias = op.bias; p.k = op.k; p.stride = op.stride; p.dil = op.dil; p.act = op.act; p.B = op.in.B;
  MYOLO_REQUIRE(op.Ci_pad % 8 == 0 && op.in.ctot % (op.in.dtype == MYOLO_F16 ? 8 : 4) == 0, "conv_simt: Ci_pad %d / ctot %d alignment",
                op.Ci_pad, op.in.ctot);
  MYOLO_REQUIRE(op.in.C >= op.Ci_pad, "conv_simt: input view has %d channels, packed weights expect %d", op.in.C, op.Ci_pad);
  const long warps = (long)p.B * p.Ho * p.Wo * ((p.Co + 7) / 8);
  long blocks = (warps + 7) / 8;
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (blocks < 1) blocks = 1;
  if (op.in.dtype == MYOLO_F16) MYOLO_CHECK_CUDA(launch_pdl(conv_simt_kernel<__half>, dim3((int)blocks), dim3(256), 0, stream, p));
  else MYOLO_CHECK_CUDA(launch_pdl(conv_simt_kernel<float>, dim3((int)blocks), dim3(256), 0, stream, p));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// BN fold + fp16 pack.   reference utils/torch_utils.py:182-202 (fuse_conv_and_bn)
// ------------------------------------------------------------------------------------------------
__global__ void pack_weights_kernel(const float* __restrict__ w, int co, int ci, int k, const float* gamma, const float* beta,
                                    const float* mean, const float* var, float eps, const float* bias, __half* wp, float* bp,
                                    int co_pad, int ci_pad) {
  const int taps = k * k;
  const long total = (long)co_pad * taps * ci_pad;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ci_pad);
    const int t = (int)((i / ci_pad) % taps);
    const int o = (int)(i / ((long)ci_pad * taps));
    float v = 0.f;
    if (o < co && c < ci) {
      v = w[((size_t)o * ci + c) * taps + t];
      if (gamma) v *= gamma[o] / sqrtf(var[o] + eps);
    }
    wp[i] = __float2half_rn(v);
  }
  for (int o = blockIdx.x * blockDim.x + threadIdx.x; o < co_pad; o += gridDim.x * blockDim.x) {
    float b = 0.f;
    if (o < co) {
      if (gamma) b = beta[o] - gamma[o] * mean[o] / sqrtf(var[o] + eps);
      if (bias) b += gamma ? bias[o] * gamma[o] / sqrtf(var[o] + eps) : bias[o];
    }
    bp[o] = b;
  }
}

// every weight pack of a plan in ONE launch (training repacks all fp16 copies after each optimiser step: ~280 tiny launches otherwise).
// A job is a forward pack (kind 0: [co_pad][taps][ci_pad], BN fold optional, bias vector) or a data-gradient pack (kind 1:
// W'[ci][tap'][co] = W[co][ci][taps-1-tap'], zero bias); block b handles chunk b of kPackChunk elements, jobs found by binary search
// over the chunk prefix.
__global__ void __launch_bounds__(256) pack_group_kernel(const PackJob* __restrict__ jobs, int n_jobs) {
  int lo = 0, hi = n_jobs - 1;
  const int b = blockIdx.x;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (jobs[mid].chunk0 <= b) lo = mid; else hi = mid - 1;
  }
  const PackJob j = jobs[lo];
  const int taps = j.k * j.k;
  const long total = (long)j.n_pad * taps * j.c_pad;
  const long base = (long)(b - j.chunk0) * kPackChunk;
  for (int e = threadIdx.x; e < kPackChunk; e += 256) {
    const long i = base + e;
    if (i >= total) break;
    const int c = (int)(i % j.c_pad);
    const int t = (int)((i / j.c_pad) % taps);
    const int n = (int)(i / ((long)j.c_pad * taps));
    float v = 0.f;
    if (j.kind == 0) {            // n = output channel, c = input channel
      if (n < j.co && c < j.ci) {
        v = j.w[((size_t)n * j.ci + c) * taps + t];
        if (j.gamma) v *= j.gamma[n] / sqrtf(j.var[n] + j.eps);
      }
    } else {                      // n = input channel (the data gradient's output), c = output channel
      if (n < j.ci && c < j.co) v = j.w[((size_t)c * j.ci + n) * taps + (taps - 1 - t)];
    }
    j.wp[i] = __float2half_rn(v);
  }
  if (b == j.chunk0) {
    for (int o = threadIdx.x; o < j.n_pad; o += 256) {
      float bv = 0.f;
      if (j.kind == 0 && o < j.co) {
        if (j.gamma) bv = j.beta[o] - j.gamma[o] * j.mean[o] / sqrtf(j.var[o] + j.eps);
        if (j.bias) bv += j.gamma ? j.bias[o] * j.gamma[o] / sqrtf(j.var[o] + j.eps) : j.bias[o];
      }
      j.bp[o] = bv;
    }
  }
}

int pack_group_launch(const PackJob* d_jobs, int n_jobs, int total_chunks, cudaStream_t stream) {
  if (n_jobs <= 0 || total_chunks <= 0) return 0;
  pack_group_kernel<<<total_chunks, 256, 0, stream>>>(d_jobs, n_jobs);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

int pack_conv_weights(const float* w, int co, int ci, int k, const float* gamma, const float* beta, const float* mean,
                      const float* var, float eps, const float* bias, __half* wp, float* bp, int co_pad, int ci_pad,
                      cudaStream_t stream) {
  const long total = (long)co_pad * k * k * ci_pad;
  int blocks = (int)((total + 255) / 256);
  if (blocks > 4096) blocks = 4096;
  pack_weights_kernel<<<blocks, 256, 0, stream>>>(w, co, ci, k, gamma, beta, mean, var, eps, bias, wp, bp, co_pad, ci_pad);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo
