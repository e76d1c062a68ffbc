// Shared helpers: error plumbing for the C ABI and thin wrappers over the sm_90a PTX used by the kernels.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/myolo.h"

namespace myolo {

// ------------------------------------------------------------------------------------------------
// error handling (thread-local message; negative codes returned through the C ABI)
// ------------------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern thread_local int64_t g_launch_count;
// 0 when the current device is an sm_90 part (its SM count into *sms, nullable), else MYOLO_E_NODEVICE with the reason set
int check_device(int* sms);

// NVTX ranges around every C-ABI entry point that launches work (SURVEY.md section 5): visible in nsys / ncu --nvtx, free when no tool is attached
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

#define MYOLO_CHECK_CUDA(expr)                                                                         \
  do {                                                                                                 \
    cudaError_t _e = (expr);                                                                           \
    if (_e != cudaSuccess) {                                                                           \
      ::myolo::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e));        \
      return MYOLO_E_CUDA;                                                                             \
    }                                                                                                  \
  } while (0)

#define MYOLO_REQUIRE(cond, ...)                 \
  do {                                           \
    if (!(cond)) {                               \
      ::myolo::set_error(__VA_ARGS__);           \
      return MYOLO_E_INVALID;                    \
    }                                            \
  } while (0)

#define MYOLO_LAUNCH_CHECK()                       \
  do {                                             \
    ::myolo::g_launch_count++;                     \
    MYOLO_CHECK_CUDA(cudaGetLastError());          \
  } while (0)

static inline int ceil_div(int a, int b) { return (a + b - 1) / b; }

// Programmatic dependent launch for the small kernels of the training chains (~1350 launches per step, most of them 5-15 us): the kernel may be
// scheduled while its stream predecessor is still running, which takes the ~2 us launch latency off the critical path.  A kernel launched
// through launch_pdl() MUST call pdl_enter() before it touches memory (its predecessor's output is only visible after the wait).
template <typename... KArgs, typename... Args>
static inline cudaError_t launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}
static inline int64_t align_up(int64_t a, int64_t b) { return (a + b - 1) / b * b; }

// A resolved NHWC tensor slice on the device.
struct TensorView {
  void* base;      // first element of image 0, pixel (0,0), channel c_off
  int B, H, W;     // extents
  int C;           // channels in the slice
  int ctot;        // channel pitch of the underlying buffer (elements per pixel)
  int dtype;       // MYOLO_F16 / MYOLO_F32
  __host__ __device__ size_t esize() const { return dtype == MYOLO_F16 ? 2 : 4; }
};

// ------------------------------------------------------------------------------------------------
// device-side PTX wrappers
// ------------------------------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_enter() {
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
}
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n"
      ".reg .b32 %%rx;\n"
      ".reg .pred %%px;\n"
      "     elect.sync %%rx|%%px, %1;\n"
      "@%%px mov.s32 %0, 1;\n"
      "}\n"
      : "+r"(pred)
      : "r"(0xFFFFFFFFu));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.b32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug becomes a trap (-> cudaErrorLaunchFailure) instead of a hung GPU.  No printf here: a call anywhere in a
// kernel that issues wgmma makes ptxas serialise the wgmma pipeline (C7510).
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity))
    if (++spins > (1u << 26)) __trap();
}

// ---- TMA ----
__device__ __forceinline__ void tma_prefetch_desc(const void* tmap) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tmap)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, uint64_t* bar, int c0, int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];" ::"r"(
          smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(tmap)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}
// SiLU with ONE transcendental (MUFU.EX2) per element: the reciprocal of 1+e^-v runs on the FMA pipe (integer seed + 3 Newton
// steps, ~4e-8 relative) so the conv epilogues are not bound by the 16-lane/clk SFU (two MUFU ops per output would be).
__device__ __forceinline__ float silu_f(float v) {
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  const float d = 1.0f + fminf(e, 1e30f);
  float r = __int_as_float(0x7EF311C7 - __float_as_int(d));
  r = r * fmaf(-d, r, 2.0f);
  r = r * fmaf(-d, r, 2.0f);
  r = r * fmaf(-d, r, 2.0f);
  return v * r;
}
// the same function with the reciprocal on the SFU (MUFU.RCP, 1 ulp): 5 issue slots instead of 12, but two MUFU ops.  The conv epilogue mixes
// both (every second element takes this one) so that the FP32 pipe (12 clk per warp-element on the Newton path) and the quarter-rate SFU
// (8 clk per MUFU) finish together: ~10 instead of 12 issue slots per element on layers whose epilogue is issue-bound (70 % issue-active in ncu).
__device__ __forceinline__ float silu_f_sfu(float v) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(v * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));      // e = +inf -> r = 0 -> v * 0 = -0 for finite v
  return v * r;
}
__device__ __forceinline__ float sigmoid_f(float v) { return __fdividef(1.0f, 1.0f + __expf(-v)); }
__device__ __forceinline__ float apply_act(float v, int act) {
  return act == MYOLO_ACT_SILU ? silu_f(v) : (act == MYOLO_ACT_SIGMOID ? sigmoid_f(v) : v);
}
#endif  // __CUDACC__

}  // namespace myolo
