// Convolution weight gradient on the Hopper tensor cores (wgmma, sm_90a), training row a13 of SURVEY.md section 8:
//
//     dW[co][ky][kx][ci] += sum over output pixels p of dY[p][co] * X[in(p, ky, kx)][ci]
//
// As a GEMM: D (M = co, N = ci) accumulates over K = output pixels.  Both operands live in HBM as NHWC fp16, i.e. with the GEMM's
// M / N dimension contiguous and K (pixels) strided: "MN-major" operands.  TMA loads [Kc pixels] x [64 channels] boxes (128-byte
// rows, SWIZZLE_128B); the wgmma shared-memory descriptors describe exactly that layout (8-row x 128-byte swizzle atoms, SBO = 1024
// bytes between 8-pixel groups, LBO = one box between 64-channel chunks) and the instruction marks A and B as transposed (MN-major).
//
// One CTA = (128 output channels) x (N input channels) x (one filter row ky: k taps) x (a slab of output rows):
//   warp 0             TMA producer: per pipeline stage one dY box set and k shifted X box sets (image border = TMA zero fill =
//                      padding; stride 2 through the four parity tensor maps, as in the forward kernel)
//   warpgroups 1 and 2 output channels [0, 64) and [64, 128) of the tile: k register accumulators of m64nNk16 wgmma (N <= 64 for 3x3
//                      so that 3 x N/2 accumulator registers per thread fit), then vector red.global.add into a [Co][k*k][Ci] fp32
//                      buffer; `unpack` adds that buffer into the caller's PyTorch-layout [Co][Ci][k][k] gradient and clears it.
// Split-K over row slabs gives every SM work; partial sums meet in the fp32 reductions.
#include <cuda.h>

#include "train.h"
#include "wgmma.cuh"

namespace myolo {

int encode_tensor_map(CUtensorMap* m, int rank, void* addr, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      int swizzle_bytes);   // conv_tc.cu

struct WgradTcParams {
  int B, Ho, Wo, Co, Ci, k, stride, dil;
  int Kc, steps_per_row, rows_total, rows_per_cta;
  int m_tiles, n_tiles, N, n_boxes;
  int bc, ci_pad, a_boxes;            // channels per X box (64 / 32 / 16 -> 128 / 64 / 32-byte swizzle); padded Ci of the packed buffer
  int num_stages, stage_bytes, a_bytes, b_bytes;
  float* dw_packed;
};

static constexpr int kWgThreads = 384;

// MN-major canonical layout: rows of `row_bytes` (128 / 64 / 32 = the swizzle width) per pixel, 8-pixel swizzle atoms
__device__ __forceinline__ uint64_t mn_major_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t row_bytes) {
  const uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : 3ull);
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);          // start address
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;  // leading byte offset: next channel chunk (one box)
  d |= (uint64_t)((8 * row_bytes) >> 4) << 32;       // stride byte offset: next group of 8 pixels
  d |= layout << 62;                                 // swizzle mode
  return d;
}

__device__ __forceinline__ void red_add_v2(float* addr, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(addr), "f"(a), "f"(b) : "memory");
}

template <int N, int K>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_tc_kernel(const __grid_constant__ CUtensorMap tmDy, const __grid_constant__ CUtensorMap tmX0,
                     const __grid_constant__ CUtensorMap tmX1, const __grid_constant__ CUtensorMap tmX2,
                     const __grid_constant__ CUtensorMap tmX3, const WgradTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)p.num_stages * p.stage_bytes);
  uint64_t* full = bars;
  uint64_t* empty = bars + p.num_stages;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
  // work item
  int t = blockIdx.x;
  const int ky = t % K; t /= K;
  const int n_tile = t % p.n_tiles; t /= p.n_tiles;
  const int m_tile = t;
  const int co0 = m_tile * 128, ci0 = n_tile * N;
  const int row0 = blockIdx.y * p.rows_per_cta;
  const int row1 = min(p.rows_total, row0 + p.rows_per_cta);
  const int n_steps = (row1 - row0) * p.steps_per_row;

  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");      // programmatic dependent launch: see common.cuh launch_pdl
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.num_stages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    fence_mbar_init();
    tma_prefetch_desc(&tmDy);
    tma_prefetch_desc(&tmX0);
  }
  __syncthreads();
  // dY, X and the packed accumulation buffer come from predecessor kernels: every thread waits (the epilogue's red.global.add must not
  // race a predecessor's unpack of the same buffer)
  asm volatile("griddepcontrol.wait;" ::: "memory");

  if (warp == 0) {
    // ===================== TMA producer (warp-converged; one elected lane issues) =====================
    const bool leader = elect_one();
    const int half = K / 2;
    int stage = 0;
    uint32_t phase = 0;
    for (int r = row0; r < row1; ++r) {
      const int b = r / p.Ho, oy = r - b * p.Ho;
      int iy, py = 0;
      if (p.stride == 1) iy = oy + (ky - half) * p.dil;
      else { py = (ky == 1) ? 0 : 1; iy = oy + (ky == 0 ? -1 : 0); }
      for (int st = 0; st < p.steps_per_row; ++st) {
        const int ox0 = st * p.Kc;
        mbar_wait(&empty[stage], phase ^ 1);
        __syncwarp();
        uint8_t* sa = smem + (size_t)stage * p.stage_bytes;
        if (leader) {
          // the bytes the boxes deliver: b_bytes is rounded up to the 1024-byte swizzle alignment (16 pixels x 16 channels = 512 bytes
          // per tap, layer 0 at input widths of 64 n + 32, would otherwise leave the barrier waiting for bytes that never come)
          mbar_arrive_expect_tx(&full[stage], (uint32_t)(p.a_boxes * p.Kc * 128 + K * p.n_boxes * p.Kc * p.bc * 2));
          tma_load_4d(sa, &tmDy, &full[stage], co0, ox0, oy, b);
          if (p.a_boxes == 2) tma_load_4d(sa + p.Kc * 128, &tmDy, &full[stage], co0 + 64, ox0, oy, b);
        }
        for (int kx = 0; kx < K; ++kx) {
          uint8_t* sb = sa + p.a_bytes + kx * p.b_bytes;
          int ix0, px = 0;
          if (p.stride == 1) ix0 = ox0 + (kx - half) * p.dil;
          else { px = (kx == 1) ? 0 : 1; ix0 = ox0 + (kx == 0 ? -1 : 0); }
          const int m = py * 2 + px;
          const CUtensorMap* tm = m == 0 ? &tmX0 : (m == 1 ? &tmX1 : (m == 2 ? &tmX2 : &tmX3));
          if (leader)
            for (int nb = 0; nb < p.n_boxes; ++nb) tma_load_4d(sb + nb * p.Kc * p.bc * 2, tm, &full[stage], ci0 + nb * p.bc, ix0, iy, b);
        }
        if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: output channels [64 cw, 64 cw + 64) of the tile =====================
    const int cw = (warp >> 2) - 1;
    const bool active = cw < p.a_boxes;      // the second warpgroup has no rows when Co <= 64
    const bool signaller = (threadIdx.x & 127) == 0;
    float acc[K][N / 2];
#pragma unroll
    for (int kx = 0; kx < K; ++kx)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) acc[kx][i] = 0.f;
    const uint32_t lbo_b = (uint32_t)p.Kc * p.bc * 2, rb = (uint32_t)p.bc * 2;
    const int jn = p.Kc / 16;
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int s = 0; s < n_steps; ++s) {
      mbar_wait(&full[stage], phase);
      if (active) {
        const uint32_t sa = smem_u32(smem + (size_t)stage * p.stage_bytes);
        wgmma_fence();
#pragma unroll
        for (int kx = 0; kx < K; ++kx) {
          wgmma_fence_regs(acc[kx]);
          for (int j = 0; j < jn; ++j)      // 16 pixels per instruction = two 8-pixel groups
            wgmma_f16<N, 1, 1>(acc[kx], mn_major_desc(sa + cw * p.Kc * 128 + j * 2048, (uint32_t)p.Kc * 128, 128),
                               mn_major_desc(sa + p.a_bytes + kx * p.b_bytes + j * 16 * rb, lbo_b, rb), (uint32_t)((s | j) != 0));
        }
        wgmma_commit();
        wgmma_wait<1>();                    // the previous stage's MMAs have retired
      }
      if (prev >= 0 && signaller) mbar_arrive(&empty[prev]);
      prev = stage;
      if (++stage == p.num_stages) { stage = 0; phase ^= 1; }
    }
    wgmma_wait<0>();
    if (prev >= 0 && signaller) mbar_arrive(&empty[prev]);
    if (active && n_steps > 0) {
      // fragment: row (co) 16*(warp%4) + lane/4 + 8h, columns (ci) 8j + 2*(lane%4) + {0,1} in acc[kx][4j + 2h + {0,1}]
      const int taps = K * K;
#pragma unroll
      for (int kx = 0; kx < K; ++kx) {
        wgmma_fence_regs(acc[kx]);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = co0 + cw * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
          if (co >= p.Co) continue;
          float* dst = p.dw_packed + ((size_t)co * taps + ky * K + kx) * p.ci_pad + ci0 + 2 * (lane & 3);
#pragma unroll
          for (int j = 0; j < N / 8; ++j) red_add_v2(dst + 8 * j, acc[kx][4 * j + 2 * h], acc[kx][4 * j + 2 * h + 1]);
        }
      }
    }
  }
}

// dW[co][ci][t] += packed[co][t][ci]; packed = 0
__global__ void wgrad_unpack_kernel(float* __restrict__ packed, float* __restrict__ dW, int co, int ci, int ci_pad, int taps) {
  pdl_enter();
  const long total = (long)co * ci_pad * taps;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i % ci_pad);
    const int t = (int)((i / ci_pad) % taps);
    const int o = (int)(i / ((long)ci_pad * taps));
    const float v = packed[i];
    packed[i] = 0.f;
    if (c < ci && v != 0.f) atomicAdd(dW + ((size_t)o * ci + c) * taps + t, v);   // both passes of a step may unpack concurrently
  }
}

template <int N, int K>
static cudaError_t launch_nk(const WgradTcParams& p, dim3 grid, size_t smem, cudaStream_t s, const CUtensorMap& tmDy, const CUtensorMap* tmX) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_tc_kernel<N, K>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return launch_pdl(conv_wgrad_tc_kernel<N, K>, grid, dim3(kWgThreads), smem, s, tmDy, tmX[0], tmX[1], tmX[2], tmX[3], p);
}

static cudaError_t launch_wgrad(const WgradTcParams& p, dim3 grid, size_t smem, cudaStream_t s, const CUtensorMap& tmDy, const CUtensorMap* tmX) {
  if (p.k == 1) {
    switch (p.N) {
      case 16: return launch_nk<16, 1>(p, grid, smem, s, tmDy, tmX);
      case 32: return launch_nk<32, 1>(p, grid, smem, s, tmDy, tmX);
      case 64: return launch_nk<64, 1>(p, grid, smem, s, tmDy, tmX);
      case 128: return launch_nk<128, 1>(p, grid, smem, s, tmDy, tmX);
    }
  } else {
    switch (p.N) {
      case 16: return launch_nk<16, 3>(p, grid, smem, s, tmDy, tmX);
      case 32: return launch_nk<32, 3>(p, grid, smem, s, tmDy, tmX);
      case 64: return launch_nk<64, 3>(p, grid, smem, s, tmDy, tmX);
    }
  }
  return cudaErrorInvalidValue;
}

bool conv_wgrad_tc_eligible(const TensorView& x, const TensorView& dy, int k, int stride, int dil, int co, int ci) {
  if (x.dtype != MYOLO_F16 || dy.dtype != MYOLO_F16) return false;
  if (!(k == 1 || k == 3)) return false;
  if (!((stride == 1) || (stride == 2 && k == 3 && dil == 1 && !((x.H | x.W) & 1)))) return false;
  const int cp = (ci + 15) / 16 * 16;                       // the view may carry zero-padded channels (layer 0: 12 -> 16)
  if (!(cp % 64 == 0 || cp == 32 || cp == 16) || x.C < cp || dy.C < co) return false;
  if (dy.W % 16 != 0 || (long)dy.B * dy.H * dy.W < 2048) return false;
  if (x.ctot % 8 != 0 || dy.ctot % 8 != 0) return false;
  if ((reinterpret_cast<uintptr_t>(x.base) & 15) || (reinterpret_cast<uintptr_t>(dy.base) & 15)) return false;
  return true;
}

// k == 1 with unpadded ci accumulates straight into the caller's [Co][Ci] gradient (when it is 16-byte aligned): no packed buffer
size_t conv_wgrad_packed_bytes(const float* dW, int co, int ci, int k) {
  const int cp = (ci + 15) / 16 * 16;
  const bool direct = k == 1 && cp == ci && (reinterpret_cast<uintptr_t>(dW) & 15) == 0;
  return direct ? 0 : (size_t)co * cp * k * k * sizeof(float);
}

int launch_conv_wgrad_tc(const TensorView& x, const TensorView& dy, int k, int stride, int dil, float* dW, float* dw_packed, int co, int ci,
                         int num_sms, cudaStream_t s, int32_t* tiling) {
  MYOLO_REQUIRE(conv_wgrad_tc_eligible(x, dy, k, stride, dil, co, ci) && dW, "conv_wgrad_tc: unsupported geometry");
  const int cp = (ci + 15) / 16 * 16;
  const bool direct = conv_wgrad_packed_bytes(dW, co, ci, k) == 0;
  MYOLO_REQUIRE(direct || dw_packed, "conv_wgrad_tc: packed accumulation buffer missing");
  WgradTcParams p;
  memset(&p, 0, sizeof(p));
  p.B = dy.B; p.Ho = dy.H; p.Wo = dy.W; p.Co = co; p.Ci = ci; p.k = k; p.stride = stride; p.dil = dil;
  p.Kc = dy.W % 64 == 0 ? 64 : (dy.W % 32 == 0 ? 32 : 16);
  p.ci_pad = cp;
  p.N = cp % 128 == 0 && k == 1 ? 128 : (cp % 64 == 0 ? 64 : cp);   // 3x3: three register accumulators of N/2 floats per thread
  p.bc = p.N >= 64 ? 64 : p.N;
  p.n_boxes = p.N / p.bc;
  p.a_boxes = co > 64 ? 2 : 1;                          // the second 64-channel dY box is skipped when it would be all padding
  auto geom = [&]() {
    p.a_bytes = 2 * p.Kc * 128;                         // room for both 64-channel dY boxes (the second is not loaded when Co <= 64)
    p.b_bytes = (int)align_up(p.n_boxes * p.Kc * p.bc * 2, 1024);
    p.stage_bytes = p.a_bytes + k * p.b_bytes;
  };
  geom();
  if (p.stage_bytes > 48 * 1024 && p.Kc > 32) {       // keep at least 4 stages in flight
    p.Kc = 32;
    geom();
  }
  p.num_stages = std::min(8, (200 * 1024) / p.stage_bytes);
  p.steps_per_row = p.Wo / p.Kc;
  p.rows_total = p.B * p.Ho;
  p.m_tiles = ceil_div(co, 128);
  p.n_tiles = cp / p.N;
  const int items = p.m_tiles * p.n_tiles * k;
  int slabs = std::max(1, (2 * num_sms) / items);
  const int min_rows = std::max(1, 4 / p.steps_per_row);            // at least ~4 pipeline steps per CTA
  slabs = std::min(slabs, std::max(1, p.rows_total / min_rows));
  p.rows_per_cta = ceil_div(p.rows_total, slabs);
  slabs = ceil_div(p.rows_total, p.rows_per_cta);
  p.dw_packed = direct ? dW : dw_packed;
  if (tiling) {
    tiling[0] = p.Kc; tiling[1] = p.N; tiling[2] = slabs; tiling[3] = p.rows_per_cta; tiling[4] = p.rows_total;
  }

  CUtensorMap tmDy, tmX[4];
  const int esz = 2;
  {
    uint64_t dims[4] = {(uint64_t)dy.C, (uint64_t)dy.W, (uint64_t)dy.H, (uint64_t)dy.B};
    uint64_t str[3] = {(uint64_t)dy.ctot * esz, (uint64_t)dy.W * dy.ctot * esz, (uint64_t)dy.H * dy.W * dy.ctot * esz};
    uint32_t box[4] = {64, (uint32_t)p.Kc, 1, 1};
    int rc = encode_tensor_map(&tmDy, 4, dy.base, dims, str, box, 128);
    if (rc) return rc;
  }
  if (stride == 1) {
    uint64_t dims[4] = {(uint64_t)x.C, (uint64_t)x.W, (uint64_t)x.H, (uint64_t)x.B};
    uint64_t str[3] = {(uint64_t)x.ctot * esz, (uint64_t)x.W * x.ctot * esz, (uint64_t)x.H * x.W * x.ctot * esz};
    uint32_t box[4] = {(uint32_t)p.bc, (uint32_t)p.Kc, 1, 1};
    int rc = encode_tensor_map(&tmX[0], 4, x.base, dims, str, box, p.bc * 2);
    if (rc) return rc;
    tmX[1] = tmX[2] = tmX[3] = tmX[0];
  } else {
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        uint64_t dims[4] = {(uint64_t)x.C, (uint64_t)x.W / 2, (uint64_t)x.H / 2, (uint64_t)x.B};
        uint64_t str[3] = {(uint64_t)2 * x.ctot * esz, (uint64_t)2 * x.W * x.ctot * esz, (uint64_t)x.H * x.W * x.ctot * esz};
        uint32_t box[4] = {(uint32_t)p.bc, (uint32_t)p.Kc, 1, 1};
        void* base = reinterpret_cast<__half*>(x.base) + ((size_t)py * x.W + px) * x.ctot;
        int rc = encode_tensor_map(&tmX[py * 2 + px], 4, base, dims, str, box, p.bc * 2);
        if (rc) return rc;
      }
  }
  const int smem = p.num_stages * p.stage_bytes + 1024 /*alignment*/ + 256 /*barriers*/;
  MYOLO_CHECK_CUDA(launch_wgrad(p, dim3(items, slabs), (size_t)smem, s, tmDy, tmX));
  MYOLO_LAUNCH_CHECK();
  if (!direct) {
    MYOLO_CHECK_CUDA(launch_pdl(wgrad_unpack_kernel, dim3(std::min(num_sms * 8, ceil_div(co * cp * k * k, 256))), dim3(256), 0, s, dw_packed, dW, co, ci,
                                cp, k * k));
    MYOLO_LAUNCH_CHECK();
  }
  return 0;
}

}  // namespace myolo
