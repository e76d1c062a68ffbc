// Device-side pre-process (SURVEY.md section 8f rank 1): letterbox (cv2.resize INTER_LINEAR + constant border 114) fused with
// BGR->RGB, HWC->CHW and the uint8 -> fp16/fp32 /255 conversion - the step right before Model.forward (reference
// utils/datasets.py:818-848 `letterbox`, :185-189 LoadImages, detect.py:135-137).  Integer work: bit exact with OpenCV's 8-bit path
// (11-bit fixed-point coefficients, two-pass rounding; exact 2x down-scaling = 2x2 area mean); parity: tests/test_gpu_pre.py.
// HBM bound: reads <= 4 source pixels per output pixel (L1/L2 absorb the overlap), writes the output once.
#include "kernels.h"

namespace myolo {

struct LetterboxParams {
  const unsigned char* src;   // (B, H0, W0, 3)
  void* dst;
  int B, H0, W0;              // source
  int rw, rh;                 // resized (un-padded) size
  int top, left;              // border offsets
  int H, W;                   // output size
  double scale_x, scale_y;    // 1 / (rw / W0), 1 / (rh / H0)   (computed on the host exactly as cv2 does)
  int mode;                   // 0: copy (no resize), 1: bilinear fixed point, 2: 2x2 area mean
  int out_dtype;              // MYOLO_U8 / MYOLO_F16 / MYOLO_F32 (float outputs are value / 255)
  int chw;                    // 1: (B,3,H,W) planes, 0: (B,H,W,3) interleaved
  int swap_rb;                // 1: output channel c = source channel 2 - c
  int pad[3];                 // border colour per SOURCE channel order
};

__device__ __forceinline__ void lin_coeff(int d, double scale, int n_src, bool clamp_frac, int* s0, int* s1, int* c0, int* c1) {
  // float((d + 0.5) * scale - 0.5) with the double operations kept separate (no fused multiply-add), as the host code computes it
  const float f = (float)__dsub_rn(__dmul_rn((double)d + 0.5, scale), 0.5);
  int s = (int)floorf(f);
  float fr = __fsub_rn(f, (float)s);
  if (clamp_frac) {                       // x direction: index and fraction are clamped at both borders
    if (s < 0) { fr = 0.f; s = 0; }
    if (s >= n_src - 1) { fr = 0.f; s = n_src - 1; }
    *s0 = s;
    *s1 = min(s + 1, n_src - 1);
  } else {                                // y direction: rows clamp, the fraction stays
    *s0 = min(max(s, 0), n_src - 1);
    *s1 = min(max(s + 1, 0), n_src - 1);
  }
  *c0 = __float2int_rn(__fmul_rn(__fsub_rn(1.0f, fr), 2048.0f));   // saturate_cast<short>(w * INTER_RESIZE_COEF_SCALE): round half even
  *c1 = __float2int_rn(__fmul_rn(fr, 2048.0f));
}

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
      const unsigned char* img = p.src + (size_t)b * p.H0 * p.W0 * 3;
      if (p.mode == 0) {
        const unsigned char* q = img + ((size_t)ry * p.W0 + rx) * 3;
        v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
      } else if (p.mode == 2) {
        const unsigned char* q0 = img + ((size_t)(2 * ry) * p.W0 + 2 * rx) * 3;
        const unsigned char* q1 = q0 + (size_t)p.W0 * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = (q0[c] + q0[3 + c] + q1[c] + q1[3 + c] + 2) >> 2;
      } else {
        int x0, x1, a0, a1, y0, y1, b0, b1;
        lin_coeff(rx, p.scale_x, p.W0, true, &x0, &x1, &a0, &a1);
        lin_coeff(ry, p.scale_y, p.H0, false, &y0, &y1, &b0, &b1);
        const unsigned char* r0 = img + (size_t)y0 * p.W0 * 3;
        const unsigned char* r1 = img + (size_t)y1 * p.W0 * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const int h0 = r0[x0 * 3 + c] * a0 + r0[x1 * 3 + c] * a1;     // horizontal pass (int32, scale 2^11)
          const int h1 = r1[x0 * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
          v[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;   // vertical pass with cv2's two-step rounding
        }
      }
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

int launch_letterbox(const unsigned char* src, int B, int H0, int W0, int rw, int rh, int top, int left, int H, int W, const int* pad3,
                     void* dst, int out_dtype, int chw, int swap_rb, cudaStream_t s) {
  MYOLO_REQUIRE(src && dst && B > 0 && H0 > 0 && W0 > 0 && rw > 0 && rh > 0 && H >= rh + top && W >= rw + left && top >= 0 && left >= 0,
                "letterbox: bad geometry (src %dx%d resized %dx%d out %dx%d offset %d,%d)", W0, H0, rw, rh, W, H, left, top);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "letterbox: output dtype");
  LetterboxParams p;
  p.src = src; p.dst = dst; p.B = B; p.H0 = H0; p.W0 = W0; p.rw = rw; p.rh = rh; p.top = top; p.left = left; p.H = H; p.W = W;
  p.scale_x = 1.0 / ((double)rw / (double)W0);
  p.scale_y = 1.0 / ((double)rh / (double)H0);
  const double eps = 2.220446049250313e-16;
  if (rw == W0 && rh == H0) p.mode = 0;
  else if (fabs(p.scale_x - 2.0) < eps && fabs(p.scale_y - 2.0) < eps) p.mode = 2;     // cv2 routes exact 2x down-scaling to INTER_AREA
  else p.mode = 1;
  p.out_dtype = out_dtype; p.chw = chw; p.swap_rb = swap_rb;
  for (int c = 0; c < 3; ++c) p.pad[c] = pad3 ? pad3[c] : 114;
  const long total = (long)B * H * W;
  letterbox_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(p);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

}  // namespace myolo
