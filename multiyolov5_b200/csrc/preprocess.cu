// Device-side pre-process (SURVEY.md section 8f rank 1): letterbox (cv2.resize INTER_LINEAR + constant border 114) fused with
// BGR->RGB, HWC->CHW and the uint8 -> fp16/fp32 /255 conversion - the step right before Model.forward (reference
// utils/datasets.py:818-848 `letterbox`, :185-189 LoadImages, detect.py:135-137).  Integer work: bit exact with OpenCV's 8-bit path
// (11-bit fixed-point coefficients, two-pass rounding; exact 2x down-scaling = 2x2 area mean); parity: tests/test_gpu_pre.py.
// HBM bound: reads <= 4 source pixels per output pixel (L1/L2 absorb the overlap), writes the output once.
#include "kernels.h"
#include "resize.cuh"

namespace myolo {

struct LetterboxParams {
  const unsigned char* src;   // (B, H0, W0, 3)
  void* dst;
  int B;
  ResizeGeom g;               // source size, scale factors and resize mode (computed on the host exactly as cv2 does)
  int rw, rh;                 // resized (un-padded) size
  int top, left;              // border offsets
  int H, W;                   // output size
  int out_dtype;              // MYOLO_U8 / MYOLO_F16 / MYOLO_F32 (float outputs are value / 255)
  int chw;                    // 1: (B,3,H,W) planes, 0: (B,H,W,3) interleaved
  int swap_rb;                // 1: output channel c = source channel 2 - c
  int pad[3];                 // border colour per SOURCE channel order
};

__global__ void letterbox_kernel(const LetterboxParams p) {
  const long total = (long)p.B * p.H * p.W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % p.W);
    const int y = (int)((i / p.W) % p.H);
    const int b = (int)(i / ((long)p.W * p.H));
    int v[3];
    const int rx = x - p.left, ry = y - p.top;
    if (rx < 0 || ry < 0 || rx >= p.rw || ry >= p.rh) {
      v[0] = p.pad[0]; v[1] = p.pad[1]; v[2] = p.pad[2];
    } else {
      resize_pixel_u8(p.src + (size_t)b * p.g.H0 * p.g.W0 * 3, p.g, rx, ry, v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int val = v[p.swap_rb ? 2 - c : c];
      const size_t o = p.chw ? (((size_t)b * 3 + c) * p.H + y) * p.W + x : (((size_t)b * p.H + y) * p.W + x) * 3 + c;
      if (p.out_dtype == MYOLO_U8) reinterpret_cast<unsigned char*>(p.dst)[o] = (unsigned char)val;
      // `img /= 255.0` on a CUDA tensor (detect.py:137): ATen multiplies by the fp32 reciprocal of a scalar divisor
      else if (p.out_dtype == MYOLO_F16) reinterpret_cast<__half*>(p.dst)[o] = __float2half_rn(__fmul_rn((float)val, 1.0f / 255.0f));
      else reinterpret_cast<float*>(p.dst)[o] = __fmul_rn((float)val, 1.0f / 255.0f);
    }
  }
}

// autoShape's ragged batch (reference models/common.py:655-658): every item letterboxed to one H x W from its own packed RGB source, CHW
// output, no channel swap.  Float outputs divide by 255 as torch's CPU `x / 255.` does (a true division, not the reciprocal product
// of the CUDA `img /= 255.0` above); fp16 rounds that fp32 quotient, as CPU half division computes in fp32.
__global__ void letterbox_items_kernel(const unsigned char* __restrict__ src, const myolo_letterbox_item* __restrict__ items, int B, int H,
                                       int W, void* dst, int out_dtype) {
  const long total = (long)B * H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int x = (int)(i % W);
    const int y = (int)((i / W) % H);
    const int b = (int)(i / ((long)W * H));
    const myolo_letterbox_item& it = items[b];
    int v[3] = {114, 114, 114};
    const int rx = x - it.left, ry = y - it.top;
    if (rx >= 0 && ry >= 0 && rx < it.rw && ry < it.rh) {
      ResizeGeom g;
      g.H0 = it.H0; g.W0 = it.W0; g.scale_x = it.scale_x; g.scale_y = it.scale_y; g.mode = it.mode;
      resize_pixel_u8(src + it.offset, g, rx, ry, v);
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const size_t o = (((size_t)b * 3 + c) * H + y) * W + x;
      if (out_dtype == MYOLO_U8) reinterpret_cast<unsigned char*>(dst)[o] = (unsigned char)v[c];
      else if (out_dtype == MYOLO_F16) reinterpret_cast<__half*>(dst)[o] = __float2half_rn(__fdiv_rn((float)v[c], 255.0f));
      else reinterpret_cast<float*>(dst)[o] = __fdiv_rn((float)v[c], 255.0f);
    }
  }
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_letterbox(const uint8_t* src, int B, int H0, int W0, int rw, int rh, int top, int left, int H, int W, const int32_t* pad3,
                               void* dst, int out_dtype, int chw, int swap_rb, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && dst && B > 0 && H0 > 0 && W0 > 0 && rw > 0 && rh > 0 && H >= rh + top && W >= rw + left && top >= 0 && left >= 0,
                "letterbox: bad geometry (src %dx%d resized %dx%d out %dx%d offset %d,%d)", W0, H0, rw, rh, W, H, left, top);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "letterbox: output dtype");
  LetterboxParams p;
  p.src = src; p.dst = dst; p.B = B; p.rw = rw; p.rh = rh; p.top = top; p.left = left; p.H = H; p.W = W;
  p.g = resize_geom(H0, W0, rh, rw);
  p.out_dtype = out_dtype; p.chw = chw; p.swap_rb = swap_rb;
  for (int c = 0; c < 3; ++c) p.pad[c] = pad3 ? pad3[c] : 114;
  const long total = (long)B * H * W;
  letterbox_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(p);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_letterbox_items(const uint8_t* src, const myolo_letterbox_item* items, int B, int H, int W, void* dst, int out_dtype,
                                     void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && items && dst && B > 0 && H > 0 && W > 0, "letterbox_items: bad arguments (B %d, out %dx%d)", B, W, H);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "letterbox_items: output dtype");
  const long total = (long)B * H * W;
  letterbox_items_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(src, items, B, H, W, dst, out_dtype);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
