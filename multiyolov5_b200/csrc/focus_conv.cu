// Layer 0 of the network in ONE kernel: Focus space-to-depth (reference models/common.py:549-550) + 3x3 Conv(12 -> Co) with folded BN +
// SiLU, straight from the caller's NCHW image (fp32 / fp16 / uint8 scaled by 1/255 like detect.py:137) to the NHWC fp16 activation.
//
// Why not the wgmma kernel: with only 12 input channels an implicit-GEMM row is 32 bytes, and TMA issues one request per row -
// the layer ends up bound by the TMA row rate, 4x above its HBM roofline (profiles/README.md).  Here a CTA converts the raw halo
// (20 x 132 x 3 pixels for an 8 x 64 output tile) ONCE into a space-to-depth fp16 tile in shared memory and feeds legacy
// mma.sync.m16n8k16 (K = 9 taps x 16 padded channels) from it with ldmatrix; the layer is memory bound (14.5 GFLOP vs 201 MB per
// batch-16 step), so HMMA throughput is irrelevant and the input is read from HBM exactly once.
#include "kernels.h"

namespace myolo {

static constexpr int kFcTileH = 8, kFcTileW = 64;            // output pixels per CTA: 8 rows (one per warp) x 64 columns
static constexpr int kFcHaloW = kFcTileW + 2, kFcHaloH = kFcTileH + 2;

// two horizontally adjacent raw pixels (columns 2*sx, 2*sx+1 are contiguous and 2-element aligned) -> fp32 in [0,1]
template <typename T> __device__ __forceinline__ float2 fc_load2(const T* p);
template <> __device__ __forceinline__ float2 fc_load2<float>(const float* p) { return __ldg(reinterpret_cast<const float2*>(p)); }
template <> __device__ __forceinline__ float2 fc_load2<__half>(const __half* p) {
  const __half2 h = __ldg(reinterpret_cast<const __half2*>(p));
  return __half22float2(h);
}
template <> __device__ __forceinline__ float2 fc_load2<uint8_t>(const uint8_t* p) {
  const uchar2 u = __ldg(reinterpret_cast<const uchar2*>(p));
  return make_float2((float)u.x / 255.0f, (float)u.y / 255.0f);    // detect.py:137
}

__device__ __forceinline__ void ldmatrix_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

// NT = Co / 8 (4 for yolov5s: Co 32, 6 for yolov5m: Co 48)
template <typename T, int NT>
__global__ void __launch_bounds__(256) focus_conv_kernel(const T* __restrict__ x, int B, int H, int W, const __half* __restrict__ wp,
                                                         const float* __restrict__ bias, TensorView out) {
  // s2d halo tile [10][66][16 halves] (32-byte rows), weights [Co][144 halves]
  __shared__ __align__(16) __half s_in[kFcHaloH * kFcHaloW * 16];
  __shared__ __align__(16) __half s_w[NT * 8 * 152];   // row pitch 152 halves (304 B): conflict-free ldmatrix rows
  const int Ho = H / 2, Wo = W / 2;
  const int tiles_x = (Wo + kFcTileW - 1) / kFcTileW;
  const int tx = blockIdx.x % tiles_x, ty = blockIdx.x / tiles_x, b = blockIdx.y;
  const int ox0 = tx * kFcTileW, oy0 = ty * kFcTileH;

  for (int i = threadIdx.x; i < NT * 8 * 18; i += blockDim.x) {      // 18 x 16-byte units per 144-half weight row
    const int n = i / 18, u = i - n * 18;
    reinterpret_cast<uint4*>(s_w + n * 152)[u] = __ldg(reinterpret_cast<const uint4*>(wp + n * 144) + u);
  }
  // space-to-depth conversion of the halo: channel = g*3 + c, g = (dy,dx) in order (0,0),(1,0),(0,1),(1,1); 12..15 zero
  for (int i = threadIdx.x; i < kFcHaloH * kFcHaloW; i += blockDim.x) {
    const int hy = i / kFcHaloW, hx = i - hy * kFcHaloW;
    const int sy = oy0 - 1 + hy, sx = ox0 - 1 + hx;
    __align__(16) __half v[16];
    if (sy >= 0 && sy < Ho && sx >= 0 && sx < Wo) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const T* p = x + (((size_t)b * 3 + c) * H + 2 * sy) * W + 2 * sx;
        const float2 r0 = fc_load2<T>(p), r1 = fc_load2<T>(p + W);
        v[0 * 3 + c] = __float2half_rn(r0.x);
        v[2 * 3 + c] = __float2half_rn(r0.y);
        v[1 * 3 + c] = __float2half_rn(r1.x);
        v[3 * 3 + c] = __float2half_rn(r1.y);
      }
#pragma unroll
      for (int c = 12; c < 16; ++c) v[c] = __float2half_rn(0.f);
    } else {
#pragma unroll
      for (int c = 0; c < 16; ++c) v[c] = __float2half_rn(0.f);
    }
    // the two 16-byte channel halves of a pixel are swapped on every other group of 4 pixels: ldmatrix (8 rows, 32-byte pitch)
    // then touches all 32 banks exactly once
    uint4* d = reinterpret_cast<uint4*>(s_in + (size_t)i * 16);
    const int swz = (hx >> 2) & 1;
    d[swz] = reinterpret_cast<uint4*>(v)[0];
    d[swz ^ 1] = reinterpret_cast<uint4*>(v)[1];
  }
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;   // warp = output row inside the tile
  float acc[4][NT][4];
#pragma unroll
  for (int m = 0; m < 4; ++m)
#pragma unroll
    for (int n = 0; n < NT; ++n)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[m][n][e] = 0.f;

  const uint32_t s_in_u = smem_u32(s_in), s_w_u = smem_u32(s_w);
  // ldmatrix row providers: A: lane -> pixel (lane & 15), k half (lane >> 4); B: lane -> n row (lane & 7) + 8*((lane >> 4) & 1), k half ((lane >> 3) & 1)
  const int a_pix = lane & 15, a_kh = lane >> 4;
  const int b_n = (lane & 7) + ((lane >> 4) << 3), b_kh = (lane >> 3) & 1;
#pragma unroll
  for (int t = 0; t < 9; ++t) {
    const int ky = t / 3, kx = t % 3;
    uint32_t bf[NT][2];
#pragma unroll
    for (int n2 = 0; n2 < NT / 2; ++n2) {
      const uint32_t addr = s_w_u + (((n2 * 16 + b_n) * 152) + t * 16 + b_kh * 8) * 2;
      ldmatrix_x4(addr, bf[2 * n2][0], bf[2 * n2][1], bf[2 * n2 + 1][0], bf[2 * n2 + 1][1]);
    }
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int hx = m * 16 + a_pix + kx, hy = warp + ky;
      const uint32_t addr = s_in_u + ((hy * kFcHaloW + hx) * 16 + (a_kh ^ ((hx >> 2) & 1)) * 8) * 2;
      uint32_t a0, a1, a2, a3;
      ldmatrix_x4(addr, a0, a1, a2, a3);
#pragma unroll
      for (int n = 0; n < NT; ++n) mma_16816(acc[m][n], a0, a1, a2, a3, bf[n][0], bf[n][1]);
    }
  }

  // epilogue: bias + SiLU -> fp16 NHWC.  C fragment: rows lane/4 and lane/4+8, channels 8n + 2*(lane%4) + {0,1}
  const int oy = oy0 + warp;
  if (oy >= Ho) return;
  const int q = lane & 3, cq = q * 2, rq = lane >> 2;
  float bv[NT][2];
#pragma unroll
  for (int n = 0; n < NT; ++n) { bv[n][0] = __ldg(bias + n * 8 + cq); bv[n][1] = __ldg(bias + n * 8 + cq + 1); }
#pragma unroll
  for (int m = 0; m < 4; ++m) {
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const int ox = ox0 + m * 16 + rq + hrow * 8;
      __half* op = reinterpret_cast<__half*>(out.base) + (((size_t)b * Ho + oy) * Wo + min(ox, Wo - 1)) * out.ctot;
      uint32_t h[NT];
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const __half2 v = __floats2half2_rn(silu_f(acc[m][n][hrow * 2 + 0] + bv[n][0]), silu_f(acc[m][n][hrow * 2 + 1] + bv[n][1]));
        h[n] = *reinterpret_cast<const uint32_t*>(&v);
      }
      if (NT == 4) {
        // the 4 lanes of a quad hold channels {2q,2q+1} of each 8-channel group: transpose so that lane q owns all 8 channels of
        // group q and can write them with ONE 16-byte store.  Round t: lane sends h[(q+t)&3], lane q receives from lane (q-t)&3.
        uint32_t r[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const int si = (q + t) & 3;
          const uint32_t send = si == 0 ? h[0] : (si == 1 ? h[1] : (si == 2 ? h[2] : h[3]));
          const uint32_t got = __shfl_sync(0xffffffffu, send, (lane & ~3) | ((q - t) & 3));
          const int from = (q - t) & 3;     // got = h_from[q] = channels 8q + 2*from, +1
          if (from == 0) r[0] = got; else if (from == 1) r[1] = got; else if (from == 2) r[2] = got; else r[3] = got;
        }
        if (ox < Wo) *reinterpret_cast<uint4*>(op + q * 8) = make_uint4(r[0], r[1], r[2], r[3]);
      } else if (ox < Wo) {
#pragma unroll
        for (int n = 0; n < NT; ++n) *reinterpret_cast<uint32_t*>(op + n * 8 + cq) = h[n];
      }
    }
  }
}

int launch_focus_conv(const void* x, int x_dtype, int B, int H, int W, const __half* wp, const float* bias, int co, const TensorView& out,
                      cudaStream_t s) {
  MYOLO_REQUIRE(H % 2 == 0 && W % 2 == 0 && out.H == H / 2 && out.W == W / 2 && out.dtype == MYOLO_F16 && out.C == co,
                "focus_conv: bad output view");
  MYOLO_REQUIRE(co == 32 || co == 48, "focus_conv: Co must be 32 or 48 (got %d)", co);
  const dim3 grid(ceil_div(W / 2, kFcTileW) * ceil_div(H / 2, kFcTileH), B);
#define FC_LAUNCH(T, NT) focus_conv_kernel<T, NT><<<grid, 256, 0, s>>>((const T*)x, B, H, W, wp, bias, out)
  if (co == 32) {
    if (x_dtype == MYOLO_F32) FC_LAUNCH(float, 4);
    else if (x_dtype == MYOLO_F16) FC_LAUNCH(__half, 4);
    else if (x_dtype == MYOLO_U8) FC_LAUNCH(uint8_t, 4);
    else MYOLO_REQUIRE(false, "focus_conv: unsupported dtype %d", x_dtype);
  } else {
    if (x_dtype == MYOLO_F32) FC_LAUNCH(float, 6);
    else if (x_dtype == MYOLO_F16) FC_LAUNCH(__half, 6);
    else if (x_dtype == MYOLO_U8) FC_LAUNCH(uint8_t, 6);
    else MYOLO_REQUIRE(false, "focus_conv: unsupported dtype %d", x_dtype);
  }
#undef FC_LAUNCH
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo
