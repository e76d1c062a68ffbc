// HBM-bound kernels of the path: layout/boundary conversion, pooling pyramids, bilinear/nearest resampling, Detect decode,
// seg-logit upsample (+argmax).  All are coalesced 16-byte-vector kernels over NHWC fp16 slices; none of this work is
// reshaped into GEMMs.
#include "kernels.h"

namespace myolo {

static inline int grid_for(long items, int block, int max_blocks = 132 * 32) {
  long b = (items + block - 1) / block;
  if (b > max_blocks) b = max_blocks;
  if (b < 1) b = 1;
  return (int)b;
}

__device__ __forceinline__ __half* vptr(const TensorView& v, int b, int y, int x) {
  return reinterpret_cast<__half*>(v.base) + (((size_t)b * v.H + y) * v.W + x) * v.ctot;
}
__device__ __forceinline__ float* vptr_f(const TensorView& v, int b, int y, int x) {
  return reinterpret_cast<float*>(v.base) + (((size_t)b * v.H + y) * v.W + x) * v.ctot;
}


// Elementwise NHWC kernels use a 3-D grid (x-chunk, y, image): no per-element div/mod chains, only x = i / nv.
struct RowIdx { int b, y, x, v; bool ok; };
__device__ __forceinline__ RowIdx row_index(int W, int nv) {
  RowIdx r;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  r.b = blockIdx.z;
  r.y = blockIdx.y;
  r.x = i / nv;
  r.v = i - r.x * nv;
  r.ok = r.x < W;
  return r;
}
static inline dim3 row_grid(const TensorView& out, int nv) { return dim3(ceil_div(out.W * nv, 256), out.H, out.B); }

// ------------------------------------------------------------------------------------------------
// input: NCHW image -> Focus space-to-depth NHWC fp16 (12 channels, zero padded to the view's 16)
//   channel = g*3 + c with g enumerating (dy,dx) = (0,0),(1,0),(0,1),(1,1)  [reference models/common.py:550]
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float to_unit(T v);
template <> __device__ __forceinline__ float to_unit<float>(float v) { return v; }
template <> __device__ __forceinline__ float to_unit<__half>(__half v) { return __half2float(v); }
template <> __device__ __forceinline__ float to_unit<uint8_t>(uint8_t v) { return (float)v / 255.0f; }  // detect.py:137

template <typename T>
__global__ void input_focus_kernel(const T* __restrict__ x, int B, int H, int W, TensorView out) {
  const int Ho = H / 2, Wo = W / 2;
  const long total = (long)B * Ho * Wo;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int ox = (int)(i % Wo);
    const int oy = (int)((i / Wo) % Ho);
    const int b = (int)(i / ((long)Wo * Ho));
    __align__(16) __half v[16];
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const T* p = x + (((size_t)b * 3 + c) * H + 2 * oy) * W + 2 * ox;
      v[0 * 3 + c] = __float2half_rn(to_unit<T>(p[0]));
      v[2 * 3 + c] = __float2half_rn(to_unit<T>(p[1]));
      v[1 * 3 + c] = __float2half_rn(to_unit<T>(p[W]));
      v[3 * 3 + c] = __float2half_rn(to_unit<T>(p[W + 1]));
    }
#pragma unroll
    for (int c = 12; c < 16; ++c) v[c] = __float2half_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(vptr(out, b, oy, ox));
    o[0] = reinterpret_cast<uint4*>(v)[0];
    o[1] = reinterpret_cast<uint4*>(v)[1];
  }
}

int launch_input_focus(const void* x, int x_dtype, int B, int H, int W, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(out.C == 16 && out.dtype == MYOLO_F16 && out.H == H / 2 && out.W == W / 2 && H % 2 == 0 && W % 2 == 0,
                "input_focus: bad output view");
  const long total = (long)B * (H / 2) * (W / 2);
  const int g = grid_for(total, 256);
  if (x_dtype == MYOLO_F32) input_focus_kernel<float><<<g, 256, 0, s>>>((const float*)x, B, H, W, out);
  else if (x_dtype == MYOLO_F16) input_focus_kernel<__half><<<g, 256, 0, s>>>((const __half*)x, B, H, W, out);
  else if (x_dtype == MYOLO_U8) input_focus_kernel<uint8_t><<<g, 256, 0, s>>>((const uint8_t*)x, B, H, W, out);
  else MYOLO_REQUIRE(false, "input_focus: unsupported dtype %d", x_dtype);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// nearest x2 (yaml layers 11, 15)
// ------------------------------------------------------------------------------------------------
__global__ void upsample_nearest2x_kernel(TensorView in, TensorView out) {
  pdl_enter();
  const RowIdx r = row_index(out.W, out.C / 8);
  if (!r.ok) return;
  const uint4 val = __ldg(reinterpret_cast<const uint4*>(vptr(in, r.b, r.y >> 1, r.x >> 1)) + r.v);
  reinterpret_cast<uint4*>(vptr(out, r.b, r.y, r.x))[r.v] = val;
}
int launch_upsample_nearest2x(const TensorView& in, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(out.H == 2 * in.H && out.W == 2 * in.W && in.C == out.C && in.C % 8 == 0 && in.ctot % 8 == 0 && out.ctot % 8 == 0,
                "upsample_nearest2x: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(upsample_nearest2x_kernel, row_grid(out, out.C / 8), dim3(256), 0, s, in, out));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// SPP: three cascaded 5x5 stride-1 "same" max pools == maxpool 5 / 9 / 13 (max is idempotent over window unions)
// one CTA per (image, 8-channel vector); the whole H x W map of that vector lives in shared memory.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint4 hmax8(uint4 a, uint4 b) {
  uint4 r;
  __half2* rr = reinterpret_cast<__half2*>(&r);
  const __half2* aa = reinterpret_cast<const __half2*>(&a);
  const __half2* bb = reinterpret_cast<const __half2*>(&b);
#pragma unroll
  for (int i = 0; i < 4; ++i) rr[i] = __hmax2(aa[i], bb[i]);
  return r;
}

__global__ void spp_pool_kernel(TensorView in, TensorView out, int n_cascade) {
  pdl_enter();
  extern __shared__ uint4 spp_smem[];
  const int HW = in.H * in.W;
  uint4* cur = spp_smem;
  uint4* tmp = spp_smem + HW;
  const int nv = in.C / 8;
  const int b = blockIdx.x / nv, v = blockIdx.x % nv;
  for (int i = threadIdx.x; i < HW; i += blockDim.x)
    cur[i] = __ldg(reinterpret_cast<const uint4*>(vptr(in, b, i / in.W, i % in.W)) + v);
  __syncthreads();
  for (int stage = 0; stage < n_cascade; ++stage) {
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
      const int y = i / in.W, x = i % in.W;
      uint4 m = cur[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        const int xx = x + d;
        if (d != 0 && xx >= 0 && xx < in.W) m = hmax8(m, cur[y * in.W + xx]);
      }
      tmp[i] = m;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < HW; i += blockDim.x) {
      const int y = i / in.W, x = i % in.W;
      uint4 m = tmp[i];
#pragma unroll
      for (int d = -2; d <= 2; ++d) {
        const int yy = y + d;
        if (d != 0 && yy >= 0 && yy < in.H) m = hmax8(m, tmp[yy * in.W + x]);
      }
      // output slice `stage` sits stage*C channels after the first output slice
      reinterpret_cast<uint4*>(vptr(out, b, y, x) + stage * in.C)[v] = m;
      cur[i] = m;  // each thread rewrites only the element it owns in this pass; readers of `cur` are behind the barrier
    }
    __syncthreads();
  }
}
// large maps (the Base head pools the 1/8-resolution map): plain 5x5 stride-1 max from global memory, one launch per cascade level
__global__ void maxpool5_nhwc_kernel(TensorView in, TensorView out) {
  const RowIdx r = row_index(out.W, out.C / 8);
  if (!r.ok) return;
  uint4 m = __ldg(reinterpret_cast<const uint4*>(vptr(in, r.b, r.y, r.x)) + r.v);
#pragma unroll
  for (int dy = -2; dy <= 2; ++dy) {
    const int yy = r.y + dy;
    if (yy < 0 || yy >= in.H) continue;
#pragma unroll
    for (int dx = -2; dx <= 2; ++dx) {
      const int xx = r.x + dx;
      if (xx < 0 || xx >= in.W || (dx == 0 && dy == 0)) continue;
      m = hmax8(m, __ldg(reinterpret_cast<const uint4*>(vptr(in, r.b, yy, xx)) + r.v));
    }
  }
  reinterpret_cast<uint4*>(vptr(out, r.b, r.y, r.x))[r.v] = m;
}

int launch_spp_pool(const TensorView& in, const TensorView& out5, int n_cascade, cudaStream_t s) {
  MYOLO_REQUIRE(in.C % 8 == 0 && in.ctot % 8 == 0 && out5.ctot % 8 == 0 && in.H == out5.H && in.W == out5.W, "spp_pool: bad views");
  const size_t smem = (size_t)in.H * in.W * 16 * 2;
  if (smem > 200 * 1024) {
    TensorView src = in;
    for (int st = 0; st < n_cascade; ++st) {
      TensorView dst = out5;
      dst.C = in.C;
      dst.base = reinterpret_cast<__half*>(out5.base) + (size_t)st * in.C;
      maxpool5_nhwc_kernel<<<row_grid(dst, dst.C / 8), 256, 0, s>>>(src, dst);
      MYOLO_LAUNCH_CHECK();
      src = dst;
    }
    return 0;
  }
  static bool attr = false;
  if (!attr) {
    MYOLO_CHECK_CUDA(cudaFuncSetAttribute(spp_pool_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    attr = true;
  }
  MYOLO_CHECK_CUDA(launch_pdl(spp_pool_kernel, dim3(in.B * (in.C / 8)), dim3(256), (size_t)smem, s, in, out5, n_cascade));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// bilinear, align_corners=True, NHWC fp16 -> NHWC fp16 slice (ATen upsample_bilinear2d index math)
// ------------------------------------------------------------------------------------------------
struct Lerp { int i0, i1; float l0, l1; };
__device__ __forceinline__ Lerp lerp_axis(int dst, int n_in, int n_out) {
  const float scale = n_out > 1 ? (float)(n_in - 1) / (float)(n_out - 1) : 0.f;
  const float src = __fmul_rn(scale, (float)dst);
  Lerp r;
  r.i0 = min((int)src, n_in - 1);
  r.i1 = r.i0 + (r.i0 < n_in - 1 ? 1 : 0);
  r.l1 = __fsub_rn(src, (float)r.i0);
  r.l0 = __fsub_rn(1.0f, r.l1);
  return r;
}
// exact ATen order, no FMA contraction: lh0*(lw0*a + lw1*b) + lh1*(lw0*c + lw1*d)
__device__ __forceinline__ float bilerp(float a, float b, float c, float d, const Lerp& ly, const Lerp& lx) {
  const float top = __fadd_rn(__fmul_rn(lx.l0, a), __fmul_rn(lx.l1, b));
  const float bot = __fadd_rn(__fmul_rn(lx.l0, c), __fmul_rn(lx.l1, d));
  return __fadd_rn(__fmul_rn(ly.l0, top), __fmul_rn(ly.l1, bot));
}

// kPpt consecutive output pixels of one 8-channel vector per thread: the row interpolation, the scale divisions and the index arithmetic are
// shared, a source column that serves two neighbouring outputs is loaded once (same arithmetic per output: results are bit-identical)
static constexpr int kBilPpt = 4;
__device__ __forceinline__ Lerp lerp_axis_s(int dst, int n_in, float scale) {
  const float src = __fmul_rn(scale, (float)dst);
  Lerp r;
  r.i0 = min((int)src, n_in - 1);
  r.i1 = r.i0 + (r.i0 < n_in - 1 ? 1 : 0);
  r.l1 = __fsub_rn(src, (float)r.i0);
  r.l0 = __fsub_rn(1.0f, r.l1);
  return r;
}
__device__ __forceinline__ void bilinear_nhwc_body4(const TensorView& in, const TensorView& out, int b, int y) {
  const int nv = out.C / 8;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int xg = i / nv, v = i - xg * nv;
  const int x0 = xg * kBilPpt;
  if (x0 >= out.W) return;
  const float sy = out.H > 1 ? (float)(in.H - 1) / (float)(out.H - 1) : 0.f;
  const float sx = out.W > 1 ? (float)(in.W - 1) / (float)(out.W - 1) : 0.f;
  const Lerp ly = lerp_axis_s(y, in.H, sy);
  const uint4* top = reinterpret_cast<const uint4*>(vptr(in, b, ly.i0, 0)) + v;
  const uint4* bot = reinterpret_cast<const uint4*>(vptr(in, b, ly.i1, 0)) + v;
  const int cstride = in.ctot / 8;                    // uint4 units between neighbouring pixels
  uint4* dst = reinterpret_cast<uint4*>(vptr(out, b, y, x0)) + v;
  const int ostride = out.ctot / 8;
  int ca = -1, cb = -1;                                // cached source columns
  uint4 ta, ba, tb, bb;
  ta = ba = tb = bb = make_uint4(0, 0, 0, 0);
#pragma unroll
  for (int p = 0; p < kBilPpt; ++p) {
    if (x0 + p >= out.W) break;
    const Lerp lx = lerp_axis_s(x0 + p, in.W, sx);
    if (lx.i0 != ca) {
      if (lx.i0 == cb) { ca = cb; ta = tb; ba = bb; }
      else { ca = lx.i0; ta = __ldg(top + (size_t)ca * cstride); ba = __ldg(bot + (size_t)ca * cstride); }
    }
    if (lx.i1 != cb) {
      if (lx.i1 == ca) { cb = ca; tb = ta; bb = ba; }
      else { cb = lx.i1; tb = __ldg(top + (size_t)cb * cstride); bb = __ldg(bot + (size_t)cb * cstride); }
    }
    const __half* ha = reinterpret_cast<const __half*>(&ta);
    const __half* hb = reinterpret_cast<const __half*>(&tb);
    const __half* hc = reinterpret_cast<const __half*>(&ba);
    const __half* hd = reinterpret_cast<const __half*>(&bb);
    uint4 o;
    __half* ho = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int k = 0; k < 8; ++k)
      ho[k] = __float2half_rn(bilerp(__half2float(ha[k]), __half2float(hb[k]), __half2float(hc[k]), __half2float(hd[k]), ly, lx));
    dst[(size_t)p * ostride] = o;
  }
}
static inline dim3 row_grid4(const TensorView& out, int nv) { return dim3(ceil_div(ceil_div(out.W, kBilPpt) * nv, 256), out.H, out.B); }
__global__ void bilinear_nhwc_kernel(TensorView in, TensorView out) {
  pdl_enter(); bilinear_nhwc_body4(in, out, blockIdx.z, blockIdx.y); }
// up to 4 independent resamplings with identical output extents in ONE launch (the four levels of PyramidPooling): blockIdx.y = level*H + y
struct BilinearGroup { TensorView in[4], out[4]; int n; };
__global__ void bilinear_nhwc_group_kernel(BilinearGroup g) {
  pdl_enter();
  const int H = g.out[0].H;
  const int level = blockIdx.y / H;
  bilinear_nhwc_body4(g.in[level], g.out[level], blockIdx.z, blockIdx.y - level * H);
}
int launch_bilinear_nhwc_group(const TensorView* in, const TensorView* out, int n, cudaStream_t s) {
  MYOLO_REQUIRE(n >= 1 && n <= 4, "bilinear_nhwc_group: %d members", n);
  BilinearGroup g;
  g.n = n;
  for (int i = 0; i < n; ++i) {
    MYOLO_REQUIRE(in[i].C == out[i].C && in[i].C % 8 == 0 && in[i].ctot % 8 == 0 && out[i].ctot % 8 == 0 && in[i].dtype == MYOLO_F16 &&
                      out[i].dtype == MYOLO_F16 && out[i].H == out[0].H && out[i].W == out[0].W && out[i].C == out[0].C && out[i].B == out[0].B,
                  "bilinear_nhwc_group: member %d does not match", i);
    g.in[i] = in[i];
    g.out[i] = out[i];
  }
  dim3 grid = row_grid4(out[0], out[0].C / 8);
  grid.y *= n;
  MYOLO_CHECK_CUDA(launch_pdl(bilinear_nhwc_group_kernel, grid, dim3(256), 0, s, g));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
int launch_bilinear_nhwc(const TensorView& in, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(in.C == out.C && in.C % 8 == 0 && in.ctot % 8 == 0 && out.ctot % 8 == 0 && in.dtype == MYOLO_F16 &&
                    out.dtype == MYOLO_F16,
                "bilinear_nhwc: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(bilinear_nhwc_kernel, row_grid4(out, out.C / 8), dim3(256), 0, s, in, out));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// adaptive average pooling in two deterministic stages.
//   stage 1: fp32 sums over "atoms" = cells of the grid formed by the union of all bin boundaries (one CTA per atom)
//   stage 2: bin = sum of a rectangle of atoms / pixel count   (AdaptiveAvgPool2d bins: start=floor(i*H/k), end=ceil((i+1)*H/k))
// ------------------------------------------------------------------------------------------------
__global__ void region_sum_kernel(TensorView in, const int* __restrict__ yb, int ny, const int* __restrict__ xb, int nx,
                                  TensorView out) {
  pdl_enter();
  __shared__ float red[256 * 8];
  const int atom = blockIdx.x % (ny * nx);
  const int b = blockIdx.x / (ny * nx);
  const int ay = atom / nx, ax = atom % nx;
  const int y0 = yb[ay], y1 = yb[ay + 1], x0 = xb[ax], x1 = xb[ax + 1];
  const int nv = in.C / 8;
  const int lanes = blockDim.x / nv;  // pixel lanes
  const int v = threadIdx.x % nv, pl = threadIdx.x / nv;
  float acc[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) acc[k] = 0.f;
  const int w = x1 - x0, npx = (y1 - y0) * w;
  if (pl < lanes) {
    for (int i = pl; i < npx; i += lanes) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(vptr(in, b, y0 + i / w, x0 + i % w)) + v);
      const __half2* h = reinterpret_cast<const __half2*>(&q);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __half22float2(h[k]);
        acc[2 * k] += f.x;
        acc[2 * k + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) red[threadIdx.x * 8 + k] = acc[k];
  __syncthreads();
  if (pl == 0) {
    for (int l = 1; l < lanes; ++l)
#pragma unroll
      for (int k = 0; k < 8; ++k) acc[k] += red[(l * nv + v) * 8 + k];
    float* o = vptr_f(out, b, ay, ax) + v * 8;
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = acc[k];
  }
}
int launch_region_sum(const TensorView& in, const int* d_yb, int ny, const int* d_xb, int nx, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(in.dtype == MYOLO_F16 && out.dtype == MYOLO_F32 && in.C % 8 == 0 && in.C / 8 <= 256 && out.C == in.C &&
                    out.H == ny && out.W == nx && in.ctot % 8 == 0,
                "region_sum: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(region_sum_kernel, dim3(in.B * ny * nx), dim3(256), 0, s, in, d_yb, ny, d_xb, nx, out));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__device__ __forceinline__ void region_combine_body(const TensorView& atoms, const int* __restrict__ bins, int nbins, const TensorView& out,
                                                    long first, long stride) {
  const long total = (long)out.B * nbins * out.C;
  for (long i = first; i < total; i += stride) {
    const int c = (int)(i % out.C);
    const int bin = (int)((i / out.C) % nbins);
    const int b = (int)(i / ((long)out.C * nbins));
    const int* bd = bins + bin * 5;
    float sum = 0.f;
    for (int ay = bd[0]; ay < bd[1]; ++ay)
      for (int ax = bd[2]; ax < bd[3]; ++ax) sum += vptr_f(atoms, b, ay, ax)[c];
    const float val = sum / (float)bd[4];
    const int oy = bin / out.W, ox = bin % out.W;
    if (out.dtype == MYOLO_F32) vptr_f(out, b, oy, ox)[c] = val;
    else vptr(out, b, oy, ox)[c] = __float2half_rn(val);
  }
}
__global__ void region_combine_kernel(TensorView atoms, const int* __restrict__ bins, int nbins, TensorView out) {
  pdl_enter();
  region_combine_body(atoms, bins, nbins, out, blockIdx.x * (long)blockDim.x + threadIdx.x, (long)gridDim.x * blockDim.x);
}
// the pooling levels of one pyramid in ONE launch: blockIdx.y = level
struct CombineGroup { const int* bins[4]; int nbins[4]; TensorView out[4]; };
__global__ void region_combine_group_kernel(TensorView atoms, CombineGroup g) {
  pdl_enter();
  const int l = blockIdx.y;
  region_combine_body(atoms, g.bins[l], g.nbins[l], g.out[l], blockIdx.x * (long)blockDim.x + threadIdx.x, (long)gridDim.x * blockDim.x);
}
int launch_region_combine_group(const TensorView& atoms, int atoms_nx, const int* const* d_bins, const int* nbins, const TensorView* out, int n,
                                cudaStream_t s) {
  MYOLO_REQUIRE(n >= 1 && n <= 4 && atoms.dtype == MYOLO_F32 && atoms.W == atoms_nx, "region_combine_group: bad arguments");
  CombineGroup g;
  long most = 0;
  for (int i = 0; i < n; ++i) {
    MYOLO_REQUIRE(out[i].H * out[i].W == nbins[i] && atoms.C == out[i].C, "region_combine_group: member %d does not match", i);
    g.bins[i] = d_bins[i]; g.nbins[i] = nbins[i]; g.out[i] = out[i];
    most = std::max(most, (long)out[i].B * nbins[i] * out[i].C);
  }
  MYOLO_CHECK_CUDA(launch_pdl(region_combine_group_kernel, dim3(grid_for(most, 256), n), dim3(256), 0, s, atoms, g));
  MYOLO_LAUNCH_CHECK();
  return 0;
}
int launch_region_combine(const TensorView& atoms, int atoms_nx, const int* d_bins, int nbins, const TensorView& out,
                          cudaStream_t s) {
  MYOLO_REQUIRE(atoms.dtype == MYOLO_F32 && out.H * out.W == nbins && atoms.C == out.C && atoms.W == atoms_nx,
                "region_combine: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(region_combine_kernel, dim3(grid_for((long)out.B * nbins * out.C, 256)), dim3(256), 0, s, atoms, d_bins, nbins, out));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// FFM: feat = feat*att + feat (in place); att is a (B,1,1,C) map (reference models/common.py:228-229)
// ------------------------------------------------------------------------------------------------
__global__ void channel_scale_kernel(TensorView feat, TensorView att) {
  pdl_enter();
  const RowIdx r = row_index(feat.W, feat.C / 8);
  if (!r.ok) return;
  uint4* ptr = reinterpret_cast<uint4*>(vptr(feat, r.b, r.y, r.x)) + r.v;
  uint4 q = *ptr;
  __half* h = reinterpret_cast<__half*>(&q);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float a = att.dtype == MYOLO_F32 ? vptr_f(att, r.b, 0, 0)[r.v * 8 + k] : __half2float(vptr(att, r.b, 0, 0)[r.v * 8 + k]);
    const float f = __half2float(h[k]);
    h[k] = __float2half_rn(fmaf(f, a, f));
  }
  *ptr = q;
}
int launch_channel_scale(const TensorView& feat, const TensorView& att, cudaStream_t s) {
  MYOLO_REQUIRE(feat.dtype == MYOLO_F16 && feat.C % 8 == 0 && feat.ctot % 8 == 0 && att.C == feat.C && att.H == 1 && att.W == 1,
                "channel_scale: bad views");
  MYOLO_CHECK_CUDA(launch_pdl(channel_scale_kernel, row_grid(feat, feat.C / 8), dim3(256), 0, s, feat, att));
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void add_kernel(TensorView a, TensorView bb, TensorView out) {
  const RowIdx r = row_index(out.W, out.C / 8);
  if (!r.ok) return;
  const uint4 qa = __ldg(reinterpret_cast<const uint4*>(vptr(a, r.b, r.y, r.x)) + r.v);
  const uint4 qb = __ldg(reinterpret_cast<const uint4*>(vptr(bb, r.b, r.y, r.x)) + r.v);
  const __half2* ha = reinterpret_cast<const __half2*>(&qa);
  const __half2* hb = reinterpret_cast<const __half2*>(&qb);
  uint4 o;
  __half2* ho = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float2 fa = __half22float2(ha[k]), fb = __half22float2(hb[k]);
    ho[k] = __floats2half2_rn(fa.x + fb.x, fa.y + fb.y);
  }
  reinterpret_cast<uint4*>(vptr(out, r.b, r.y, r.x))[r.v] = o;
}
int launch_add(const TensorView& a, const TensorView& b, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(a.C == out.C && b.C == out.C && out.C % 8 == 0 && a.H == out.H && b.H == out.H && a.W == out.W && b.W == out.W,
                "add: bad views");
  add_kernel<<<row_grid(out, out.C / 8), 256, 0, s>>>(a, b, out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

__global__ void broadcast_kernel(TensorView in, TensorView out) {
  const RowIdx r = row_index(out.W, out.C / 8);
  if (!r.ok) return;
  reinterpret_cast<uint4*>(vptr(out, r.b, r.y, r.x))[r.v] = __ldg(reinterpret_cast<const uint4*>(vptr(in, r.b, 0, 0)) + r.v);
}
int launch_broadcast(const TensorView& in, const TensorView& out, cudaStream_t s) {
  MYOLO_REQUIRE(in.C == out.C && in.H == 1 && in.W == 1 && in.dtype == MYOLO_F16 && out.C % 8 == 0, "broadcast: bad views");
  broadcast_kernel<<<row_grid(out, out.C / 8), 256, 0, s>>>(in, out);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Detect.forward (eval): view (bs,na,no,ny,nx) -> permute (bs,na,ny,nx,no); sigmoid; xy=(s*2-0.5+grid)*stride;
// wh=(s*2)^2*anchor; z = cat over levels                                     [reference models/yolo.py:211-225]
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float detect_decode_one(float v, int o, int x, int y, int a, float stride, const float* __restrict__ anchors) {
  float sg = __fdividef(1.0f, 1.0f + __expf(-v));
  if (o == 0) sg = (sg * 2.0f - 0.5f + (float)x) * stride;
  else if (o == 1) sg = (sg * 2.0f - 0.5f + (float)y) * stride;
  else if (o == 2 || o == 3) {
    const float t = sg * 2.0f;
    sg = t * t * anchors[a * 2 + (o - 2)];
  }
  return sg;
}
// grid = (chunks of W*no/4, H, B*na).  For a fixed (image, anchor, row) both outputs are contiguous over (x, o): a thread takes FOUR consecutive
// (x, o) positions - scalar reads of the head conv's fp32 NHWC rows (just written: L2), one 16-byte store each to raw and z.
template <int NO>
__global__ void detect_decode_kernel(TensorView in, int na, int no_rt, float stride, const float* __restrict__ anchors, float* raw,
                                     float* z, int z_off, int z_rows, int vec) {
  const int no = NO > 0 ? NO : no_rt;
  const int j0 = (blockIdx.x * blockDim.x + threadIdx.x) * 4;
  const int row_elems = in.W * no;
  if (j0 >= row_elems) return;
  const int y = blockIdx.y;
  const int b = blockIdx.z / na, a = blockIdx.z - b * na;
  const float* src = vptr_f(in, b, y, 0) + a * no;
  const size_t row = ((size_t)(b * na + a) * in.H + y) * in.W;
  float v[4], d[4];
  int x = j0 / no, o = j0 - x * no;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const bool ok = j0 + k < row_elems;
    v[k] = ok ? src[(size_t)x * in.ctot + o] : 0.f;
    d[k] = (z && ok) ? detect_decode_one(v[k], o, x, y, a, stride, anchors) : 0.f;
    if (++o == no) { o = 0; ++x; }
  }
  const bool full = vec && j0 + 3 < row_elems;       // rows that are not a multiple of 16 bytes (odd maps) take scalar stores
  if (raw) {
    float* p = raw + row * no + j0;
    if (full) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    else for (int k = 0; k < 4 && j0 + k < row_elems; ++k) p[k] = v[k];
  }
  if (!z) return;     // train mode: only the raw, permuted head outputs (reference models/yolo.py:225 `return x if self.training`)
  float* q = z + ((size_t)b * z_rows + z_off + ((size_t)a * in.H + y) * in.W) * no + j0;
  if (full) *reinterpret_cast<float4*>(q) = make_float4(d[0], d[1], d[2], d[3]);
  else for (int k = 0; k < 4 && j0 + k < row_elems; ++k) q[k] = d[k];
}
int launch_detect_decode(const TensorView& in, int na, int no, float stride, const float* d_anchors, float* raw, float* z,
                         int z_row_offset, int z_rows_total, cudaStream_t s) {
  MYOLO_REQUIRE(in.dtype == MYOLO_F32 && in.C >= na * no, "detect_decode: bad view");
  // 16-byte stores need (W * no) % 4 == 0 rows and 16-byte aligned bases (torch allocations are; z_row_offset * no * 4 must be too)
  const bool vec_ok = (in.W * no) % 4 == 0 && ((size_t)z_row_offset * no) % 4 == 0 && ((size_t)z_rows_total * no) % 4 == 0 &&
                      (!raw || (reinterpret_cast<uintptr_t>(raw) & 15) == 0) && (!z || (reinterpret_cast<uintptr_t>(z) & 15) == 0);
  const dim3 grid(ceil_div(ceil_div(in.W * no, 4), 128), in.H, in.B * na);
  if (no == 15) detect_decode_kernel<15><<<grid, 128, 0, s>>>(in, na, no, stride, d_anchors, raw, z, z_row_offset, z_rows_total, (int)vec_ok);
  else detect_decode_kernel<0><<<grid, 128, 0, s>>>(in, na, no, stride, d_anchors, raw, z, z_row_offset, z_rows_total, (int)vec_ok);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// final seg upsample: fp32 NHWC low-res logits (ctot-padded) -> NCHW logits and/or fused argmax (first max wins)
// one thread per output pixel; x fastest so every per-class store is a coalesced 128-byte line per warp.
// ------------------------------------------------------------------------------------------------
template <typename TOut> struct Pack4;
template <> struct Pack4<float> {
  static __device__ __forceinline__ void store(float* p, float a, float b, float c, float d) { *reinterpret_cast<float4*>(p) = make_float4(a, b, c, d); }
};
template <> struct Pack4<__half> {
  static __device__ __forceinline__ void store(__half* p, float a, float b, float c, float d) {
    uint2 u;
    *reinterpret_cast<__half2*>(&u.x) = __floats2half2_rn(a, b);
    *reinterpret_cast<__half2*>(&u.y) = __floats2half2_rn(c, d);
    *reinterpret_cast<uint2*>(p) = u;
  }
};

// One CTA = one output row segment of 4*blockDim.x pixels of one image.  While staging, the two source rows the output row
// needs are blended vertically once per (class, source column) into shared memory [class][col] (col fastest -> conflict-free);
// every thread then produces 4 consecutive pixels for all classes with 2 shared loads + 1 lerp per value and 16-byte stores
// (per class a warp writes 512 contiguous bytes).  (Vertical-then-horizontal association differs from ATen's
// horizontal-then-vertical by <= 1 ulp; the bit-exact-vs-ATen path is myolo_seg_upsample_argmax / myolo_bilinear_nchw.)
template <typename TOut> struct Pack8;       // 8 consecutive outputs with 16-byte stores
template <> struct Pack8<float> {
  static __device__ __forceinline__ void store(float* p, const float* v) {
    *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(p + 4) = make_float4(v[4], v[5], v[6], v[7]);
  }
};
template <> struct Pack8<__half> {
  static __device__ __forceinline__ void store(__half* p, const float* v) {
    uint4 u;
    __half2* h = reinterpret_cast<__half2*>(&u);
#pragma unroll
    for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(v[2 * k], v[2 * k + 1]);
    *reinterpret_cast<uint4*>(p) = u;
  }
};

// PPT consecutive pixels per thread (8 on the aligned fast path: one 16-byte store per class for fp16 logits, two for fp32; 4 otherwise);
// AMAX compiles the running arg-max in only when a class map is requested.
template <typename TOut, int PPT, bool AMAX>
__global__ void __launch_bounds__(256) seg_upsample_kernel(TensorView in, int ncls, int H, int W, TOut* seg, int64_t* amax) {
  extern __shared__ float sup_smem[];
  const int segs = (W + PPT * blockDim.x - 1) / (PPT * blockDim.x);
  const int sx = blockIdx.x % segs;
  const int y = (blockIdx.x / segs) % H;
  const int b = blockIdx.x / (segs * H);
  const int xbeg = sx * PPT * blockDim.x;
  const int xend = min(W, xbeg + PPT * (int)blockDim.x);
  const Lerp ly = lerp_axis(y, in.H, H);
  const int c0 = lerp_axis(xbeg, in.W, W).i0;
  const int c1 = lerp_axis(xend - 1, in.W, W).i1;
  const int ncol = c1 - c0 + 1;
  const int pitch = ncol | 1;                      // odd pitch: rows of different classes start in different banks
  float* sv = sup_smem;                            // [ncls][pitch] vertically blended source row
  const int c4n = (ncls + 3) / 4;
  for (int i = threadIdx.x; i < ncol * c4n; i += blockDim.x) {
    const int col = i / c4n, c4 = i - col * c4n;
    const float4 t = __ldg(reinterpret_cast<const float4*>(vptr_f(in, b, ly.i0, c0 + col)) + c4);
    const float4 u = __ldg(reinterpret_cast<const float4*>(vptr_f(in, b, ly.i1, c0 + col)) + c4);
    const float vv[4] = {fmaf(ly.l1, u.x, ly.l0 * t.x), fmaf(ly.l1, u.y, ly.l0 * t.y), fmaf(ly.l1, u.z, ly.l0 * t.z),
                         fmaf(ly.l1, u.w, ly.l0 * t.w)};
    float* d = sv + col;
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (c4 * 4 + k < ncls) d[(c4 * 4 + k) * pitch] = vv[k];
  }
  __syncthreads();
  const int x0 = xbeg + PPT * threadIdx.x;
  if (x0 >= W) return;
  int i0[PPT], i1[PPT];
  float l0[PPT], l1[PPT];
#pragma unroll
  for (int j = 0; j < PPT; ++j) {
    const Lerp lx = lerp_axis(min(x0 + j, W - 1), in.W, W);
    i0[j] = lx.i0 - c0; i1[j] = lx.i1 - c0; l0[j] = lx.l0; l1[j] = lx.l1;
  }
  float best[PPT];
  int bi[PPT];
#pragma unroll
  for (int j = 0; j < PPT; ++j) { best[j] = 0.f; bi[j] = 0; }
  const bool full = (x0 + PPT - 1 < W) && (W % PPT == 0);
  for (int c = 0; c < ncls; ++c) {
    const float* r = sv + c * pitch;
    float v[PPT];
#pragma unroll
    for (int j = 0; j < PPT; ++j) {
      v[j] = fmaf(l1[j], r[i1[j]], l0[j] * r[i0[j]]);
      if (AMAX && (c == 0 || v[j] > best[j])) { best[j] = v[j]; bi[j] = c; }
    }
    if (seg) {
      TOut* o = seg + (((size_t)b * ncls + c) * H + y) * W + x0;
      if (full) {
        if (PPT == 8) Pack8<TOut>::store(o, v);
        else Pack4<TOut>::store(o, v[0], v[1], v[2], v[3]);
      } else {
        for (int j = 0; j < PPT && x0 + j < W; ++j) o[j] = (TOut)v[j];
      }
    }
  }
  if (AMAX) {
    int64_t* o = amax + ((size_t)b * H + y) * W + x0;
    for (int j = 0; j < PPT && x0 + j < W; ++j) o[j] = bi[j];
  }
}
template <typename TOut>
static void launch_seg_upsample_t(const TensorView& in, int n_cls, int H, int W, TOut* seg, int64_t* argmax, size_t smem, cudaStream_t s) {
  const bool wide = (W % 8 == 0) && W >= 256 && (reinterpret_cast<uintptr_t>(seg) & 15) == 0;
  if (wide) {
    const int threads = W >= 1024 ? 128 : (W >= 512 ? 64 : 32);
    const long blocks = (long)in.B * H * ceil_div(W, 8 * threads);
    if (argmax) seg_upsample_kernel<TOut, 8, true><<<(unsigned)blocks, threads, smem, s>>>(in, n_cls, H, W, seg, argmax);
    else seg_upsample_kernel<TOut, 8, false><<<(unsigned)blocks, threads, smem, s>>>(in, n_cls, H, W, seg, argmax);
  } else {
    const int threads = W >= 1024 ? 256 : (W >= 512 ? 128 : 64);
    const long blocks = (long)in.B * H * ceil_div(W, 4 * threads);
    if (argmax) seg_upsample_kernel<TOut, 4, true><<<(unsigned)blocks, threads, smem, s>>>(in, n_cls, H, W, seg, argmax);
    else seg_upsample_kernel<TOut, 4, false><<<(unsigned)blocks, threads, smem, s>>>(in, n_cls, H, W, seg, argmax);
  }
}
int launch_seg_upsample(const TensorView& in, int n_cls, int H, int W, void* seg, int seg_dtype, int64_t* argmax, cudaStream_t s) {
  MYOLO_REQUIRE(in.dtype == MYOLO_F32 && in.ctot % 4 == 0 && in.ctot >= ((n_cls + 3) / 4) * 4, "seg_upsample: bad view");
  const size_t smem = (size_t)n_cls * ((in.W + 2) | 1) * 4;
  MYOLO_REQUIRE(smem <= 48 * 1024, "seg_upsample: source row too wide for the shared-memory kernel (%d cols x %d classes)", in.W, n_cls);
  if (seg_dtype == MYOLO_F16) launch_seg_upsample_t<__half>(in, n_cls, H, W, (__half*)seg, argmax, smem, s);
  else launch_seg_upsample_t<float>(in, n_cls, H, W, (float*)seg, argmax, smem, s);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

// ------------------------------------------------------------------------------------------------
// standalone post-process entry points on NCHW logits (detect.py:191-193)
// ------------------------------------------------------------------------------------------------
template <typename TIn, typename TOut>
__global__ void seg_argmax_nchw_kernel(const TIn* __restrict__ src, int B, int C, int h, int w, int H, int W, TOut* out) {
  const long total = (long)B * H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int b = (int)(i / ((long)W * H));
    const Lerp ly = lerp_axis(y, h, H), lx = lerp_axis(x, w, W);
    float best = 0.f;
    int bi = 0;
    for (int c = 0; c < C; ++c) {
      const TIn* pl = src + ((size_t)b * C + c) * h * w;
      float val = bilerp((float)pl[ly.i0 * w + lx.i0], (float)pl[ly.i0 * w + lx.i1], (float)pl[ly.i1 * w + lx.i0],
                         (float)pl[ly.i1 * w + lx.i1], ly, lx);
      // half logits: F.interpolate on a half tensor returns fp16 values, and the reference takes max(0) over THOSE (detect.py:191-193)
      if (sizeof(TIn) == 2) val = __half2float(__float2half_rn(val));
      if (c == 0 || val > best) { best = val; bi = c; }
    }
    out[i] = (TOut)bi;
  }
}

// same-size case of detect.py:191-193 (bilinear to the identical size is the identity): pure argmax, 4 pixels per thread,
// one 16-byte load per class plane -> C independent loads in flight per thread.
template <typename TOut>
__global__ void argmax_nchw_f32x4_kernel(const float* __restrict__ src, int B, int C, long HW, TOut* out) {
  const long n4 = (long)B * HW / 4;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n4; i += (long)gridDim.x * blockDim.x) {
    const long pix = i * 4;
    const long b = pix / HW, off = pix - b * HW;
    const float* p = src + b * C * HW + off;
    float4 best = __ldg(reinterpret_cast<const float4*>(p));
    int i0 = 0, i1 = 0, i2 = 0, i3 = 0;
#pragma unroll 6
    for (int c = 1; c < C; ++c) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(p + (size_t)c * HW));
      if (v.x > best.x) { best.x = v.x; i0 = c; }
      if (v.y > best.y) { best.y = v.y; i1 = c; }
      if (v.z > best.z) { best.z = v.z; i2 = c; }
      if (v.w > best.w) { best.w = v.w; i3 = c; }
    }
    out[pix] = (TOut)i0; out[pix + 1] = (TOut)i1; out[pix + 2] = (TOut)i2; out[pix + 3] = (TOut)i3;
  }
}

// fp16 logits (the reference's CUDA path runs model.half(), detect.py:96-103): 8 pixels per thread, one 16-byte load per class plane
// 16 pixels per thread: two independent 16-byte loads per class plane keep twice the bytes in flight (the 8-pixel version reached half the
// HBM rate of the fp32 kernel, which moves twice the bytes per thread)
template <typename TOut>
__global__ void argmax_nchw_f16x16_kernel(const __half* __restrict__ src, int B, int C, long HW, TOut* out) {
  const long n16 = (long)B * HW / 16;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n16; i += (long)gridDim.x * blockDim.x) {
    const long pix = i * 16;
    const long b = pix / HW, off = pix - b * HW;
    const __half* p = src + b * C * HW + off;
    __half2 best[8];
    unsigned char bi[16];
    {
      const uint4 v0 = __ldg(reinterpret_cast<const uint4*>(p)), v1 = __ldg(reinterpret_cast<const uint4*>(p) + 1);
      const __half2* h0 = reinterpret_cast<const __half2*>(&v0);
      const __half2* h1 = reinterpret_cast<const __half2*>(&v1);
#pragma unroll
      for (int k = 0; k < 4; ++k) { best[k] = h0[k]; best[4 + k] = h1[k]; }
#pragma unroll
      for (int k = 0; k < 16; ++k) bi[k] = 0;
    }
#pragma unroll 3
    for (int c = 1; c < C; ++c) {
      const uint4 v0 = __ldg(reinterpret_cast<const uint4*>(p + (size_t)c * HW)), v1 = __ldg(reinterpret_cast<const uint4*>(p + (size_t)c * HW) + 1);
      const __half2* h0 = reinterpret_cast<const __half2*>(&v0);
      const __half2* h1 = reinterpret_cast<const __half2*>(&v1);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const __half2 h = k < 4 ? h0[k] : h1[k - 4];
        // strict '>' per lane on the fp16 values themselves (exact: no conversion needed); first maximum wins like torch.max
        const __half2 gt = __hgt2(h, best[k]);
        if (__low2float(gt) != 0.f) { best[k] = __halves2half2(__low2half(h), __high2half(best[k])); bi[2 * k] = (unsigned char)c; }
        if (__high2float(gt) != 0.f) { best[k] = __halves2half2(__low2half(best[k]), __high2half(h)); bi[2 * k + 1] = (unsigned char)c; }
      }
    }
    if (sizeof(TOut) == 1) {
      uint4 o;
      unsigned char* ob = reinterpret_cast<unsigned char*>(&o);
#pragma unroll
      for (int k = 0; k < 16; ++k) ob[k] = bi[k];
      *reinterpret_cast<uint4*>(out + pix) = o;
    } else if (sizeof(TOut) == 8) {
#pragma unroll
      for (int k = 0; k < 8; ++k)
        reinterpret_cast<ulonglong2*>(out + pix)[k] = make_ulonglong2((unsigned long long)bi[2 * k], (unsigned long long)bi[2 * k + 1]);
    } else {
#pragma unroll
      for (int k = 0; k < 16; ++k) out[pix + k] = (TOut)bi[k];
    }
  }
}

template <typename TOut>
__global__ void argmax_nchw_f16x8_kernel(const __half* __restrict__ src, int B, int C, long HW, TOut* out) {
  const long n8 = (long)B * HW / 8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n8; i += (long)gridDim.x * blockDim.x) {
    const long pix = i * 8;
    const long b = pix / HW, off = pix - b * HW;
    const __half* p = src + b * C * HW + off;
    float best[8];
    int bi[8];
    {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p));
      const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int k = 0; k < 8; ++k) { best[k] = __half2float(h[k]); bi[k] = 0; }
    }
#pragma unroll 6
    for (int c = 1; c < C; ++c) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(p + (size_t)c * HW));
      const __half* h = reinterpret_cast<const __half*>(&v);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float f = __half2float(h[k]);
        if (f > best[k]) { best[k] = f; bi[k] = c; }
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) out[pix + k] = (TOut)bi[k];
  }
}

__global__ void bilinear_nchw_kernel(const float* __restrict__ src, int B, int C, int h, int w, int H, int W, float* dst) {
  const long total = (long)B * C * H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const long bc = i / ((long)W * H);
    const Lerp ly = lerp_axis(y, h, H), lx = lerp_axis(x, w, W);
    const float* pl = src + (size_t)bc * h * w;
    dst[i] = bilerp(pl[ly.i0 * w + lx.i0], pl[ly.i0 * w + lx.i1], pl[ly.i1 * w + lx.i0], pl[ly.i1 * w + lx.i1], ly, lx);
  }
}

__global__ void read_view_kernel(TensorView v, float* dst) {
  const long total = (long)v.B * v.C * v.H * v.W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % v.W);
    const int y = (int)((i / v.W) % v.H);
    const int c = (int)((i / ((long)v.W * v.H)) % v.C);
    const int b = (int)(i / ((long)v.W * v.H * v.C));
    dst[i] = v.dtype == MYOLO_F32 ? vptr_f(v, b, y, x)[c] : __half2float(vptr(v, b, y, x)[c]);
  }
}
int launch_read_view(const TensorView& v, float* dst, cudaStream_t s) {
  read_view_kernel<<<grid_for((long)v.B * v.C * v.H * v.W, 256), 256, 0, s>>>(v, dst);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_seg_upsample_argmax(const void* logits, int dtype, int B, int C, int h, int w, int H, int W, void* out,
                                         int out_dtype, void* stream) {
  MYOLO_REQUIRE(logits && out && B > 0 && C > 0 && h > 0 && w > 0 && H > 0 && W > 0, "seg_upsample_argmax: bad arguments");
  MYOLO_REQUIRE((dtype == MYOLO_F32 || dtype == MYOLO_F16) && (out_dtype == MYOLO_I64 || out_dtype == MYOLO_U8),
                "seg_upsample_argmax: unsupported dtype");
  cudaStream_t s = (cudaStream_t)stream;
  const int g = grid_for((long)B * H * W, 256, 132 * 64);
  if (dtype == MYOLO_F32 && H == h && W == w && ((long)H * W) % 4 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    const int g4 = grid_for((long)B * H * W / 4, 256, 132 * 32);
    if (out_dtype == MYOLO_I64) argmax_nchw_f32x4_kernel<int64_t><<<g4, 256, 0, s>>>((const float*)logits, B, C, (long)H * W, (int64_t*)out);
    else argmax_nchw_f32x4_kernel<uint8_t><<<g4, 256, 0, s>>>((const float*)logits, B, C, (long)H * W, (uint8_t*)out);
    MYOLO_LAUNCH_CHECK();
    return 0;
  }
  if (dtype == MYOLO_F16 && H == h && W == w && ((long)H * W) % 16 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0 &&
      (reinterpret_cast<uintptr_t>(out) & 15) == 0 && C <= 255) {
    const int g16 = grid_for((long)B * H * W / 16, 256, 132 * 32);
    if (out_dtype == MYOLO_I64) argmax_nchw_f16x16_kernel<int64_t><<<g16, 256, 0, s>>>((const __half*)logits, B, C, (long)H * W, (int64_t*)out);
    else argmax_nchw_f16x16_kernel<uint8_t><<<g16, 256, 0, s>>>((const __half*)logits, B, C, (long)H * W, (uint8_t*)out);
    MYOLO_LAUNCH_CHECK();
    return 0;
  }
  if (dtype == MYOLO_F16 && H == h && W == w && ((long)H * W) % 8 == 0 && (reinterpret_cast<uintptr_t>(logits) & 15) == 0) {
    const int g8 = grid_for((long)B * H * W / 8, 256, 132 * 32);
    if (out_dtype == MYOLO_I64) argmax_nchw_f16x8_kernel<int64_t><<<g8, 256, 0, s>>>((const __half*)logits, B, C, (long)H * W, (int64_t*)out);
    else argmax_nchw_f16x8_kernel<uint8_t><<<g8, 256, 0, s>>>((const __half*)logits, B, C, (long)H * W, (uint8_t*)out);
    MYOLO_LAUNCH_CHECK();
    return 0;
  }
  if (dtype == MYOLO_F32) {
    if (out_dtype == MYOLO_I64) seg_argmax_nchw_kernel<float, int64_t><<<g, 256, 0, s>>>((const float*)logits, B, C, h, w, H, W, (int64_t*)out);
    else seg_argmax_nchw_kernel<float, uint8_t><<<g, 256, 0, s>>>((const float*)logits, B, C, h, w, H, W, (uint8_t*)out);
  } else {
    if (out_dtype == MYOLO_I64) seg_argmax_nchw_kernel<__half, int64_t><<<g, 256, 0, s>>>((const __half*)logits, B, C, h, w, H, W, (int64_t*)out);
    else seg_argmax_nchw_kernel<__half, uint8_t><<<g, 256, 0, s>>>((const __half*)logits, B, C, h, w, H, W, (uint8_t*)out);
  }
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_bilinear_nchw(const float* src, int B, int C, int h, int w, int H, int W, float* dst, void* stream) {
  MYOLO_REQUIRE(src && dst && B > 0 && C > 0, "bilinear_nchw: bad arguments");
  bilinear_nchw_kernel<<<grid_for((long)B * C * H * W, 256, 132 * 64), 256, 0, (cudaStream_t)stream>>>(src, B, C, h, w, H, W, dst);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
