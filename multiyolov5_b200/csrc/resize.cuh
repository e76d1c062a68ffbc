// cv2.resize(INTER_LINEAR) of 8-bit 3-channel images, one destination pixel at a time, bit exact with OpenCV's 8-bit path: 11-bit
// fixed-point coefficients with two-pass rounding, exact 2x down-scaling routed to the 2x2 area mean as cv2 does.  Shared by the
// letterbox kernel (preprocess.cu) and the training image cache (augment.cu).  Below it, cv2.resize(INTER_AREA) down-scaling for the
// validation image cache (augment.cu), which shares the scale computation and the 2x2 mean.
#pragma once
#include <cuda_runtime.h>

#include <cmath>

namespace myolo {

// 0: copy (no resize), 1: bilinear fixed point, 2: 2x2 area mean.  scale_x / scale_y: 1 / (dst / src) in double, as cv2 computes them.
struct ResizeGeom {
  int H0, W0;
  double scale_x, scale_y;
  int mode;
};

inline ResizeGeom resize_geom(int H0, int W0, int rh, int rw) {
  ResizeGeom g;
  g.H0 = H0; g.W0 = W0;
  g.scale_x = 1.0 / ((double)rw / (double)W0);
  g.scale_y = 1.0 / ((double)rh / (double)H0);
  const double eps = 2.220446049250313e-16;
  if (rw == W0 && rh == H0) g.mode = 0;
  else if (std::fabs(g.scale_x - 2.0) < eps && std::fabs(g.scale_y - 2.0) < eps) g.mode = 2;     // cv2 routes exact 2x down-scaling to INTER_AREA
  else g.mode = 1;
  return g;
}

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

// destination pixel (rx, ry) of the resize of the HWC uint8 image `img` (g.H0 x g.W0 x 3)
__device__ __forceinline__ void resize_pixel_u8(const unsigned char* img, const ResizeGeom& g, int rx, int ry, int v[3]) {
  if (g.mode == 0) {
    const unsigned char* q = img + ((size_t)ry * g.W0 + rx) * 3;
    v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
  } else if (g.mode == 2) {
    const unsigned char* q0 = img + ((size_t)(2 * ry) * g.W0 + 2 * rx) * 3;
    const unsigned char* q1 = q0 + (size_t)g.W0 * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (q0[c] + q0[3 + c] + q1[c] + q1[3 + c] + 2) >> 2;
  } else {
    int x0, x1, a0, a1, y0, y1, b0, b1;
    lin_coeff(rx, g.scale_x, g.W0, true, &x0, &x1, &a0, &a1);
    lin_coeff(ry, g.scale_y, g.H0, false, &y0, &y1, &b0, &b1);
    const unsigned char* r0 = img + (size_t)y0 * g.W0 * 3;
    const unsigned char* r1 = img + (size_t)y1 * g.W0 * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int h0 = r0[x0 * 3 + c] * a0 + r0[x1 * 3 + c] * a1;     // horizontal pass (int32, scale 2^11)
      const int h1 = r1[x0 * 3 + c] * a0 + r1[x1 * 3 + c] * a1;
      v[c] = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;   // vertical pass with cv2's two-step rounding
    }
  }
}

// cv2.resize(INTER_AREA) of 8-bit 3-channel images, down-scaling only (load_image with augment=False).  Modes as cv2 chooses them:
// 0: copy, 2: 2x2 mean (sum + 2) >> 2, 3: other integral kx x ky block, rint(float(sum) * (1.f / (kx * ky))), 4: the general
// computeResizeAreaTab + ResizeArea_Invoker arithmetic in float32.
struct AreaGeom {
  int H0, W0;
  double scale_x, scale_y;
  int kx, ky;
  int mode;
};

inline AreaGeom area_geom(int H0, int W0, int H, int W) {
  AreaGeom g;
  g.H0 = H0; g.W0 = W0;
  g.scale_x = 1.0 / ((double)W / (double)W0);
  g.scale_y = 1.0 / ((double)H / (double)H0);
  g.kx = (int)std::lrint(g.scale_x);
  g.ky = (int)std::lrint(g.scale_y);
  const double eps = 2.220446049250313e-16;
  const bool integral = std::fabs(g.scale_x - g.kx) < eps && std::fabs(g.scale_y - g.ky) < eps;
  if (W == W0 && H == H0) g.mode = 0;
  else if (integral && g.kx == 2 && g.ky == 2) g.mode = 2;
  else if (integral) g.mode = 3;
  else g.mode = 4;
  return g;
}

// computeResizeAreaTab for destination index d of one axis, in double.  The taps are the contiguous sources s0 .. s0 + n - 1: the
// first weighs w_first when `first` (a partial leading cell), the last weighs w_last when `last`, every other one w_mid.
struct AreaTaps {
  int s0, n, first, last;
  float w_first, w_mid, w_last;
};

__device__ __forceinline__ AreaTaps area_taps(int d, double scale, int n_src) {
  const double fs1 = __dmul_rn((double)d, scale);
  const double fs2 = __dadd_rn(fs1, scale);
  const double cell = fmin(scale, __dsub_rn((double)n_src, fs1));
  const int s2 = min((int)floor(fs2), n_src - 1);
  const int s1 = min((int)ceil(fs1), s2);
  AreaTaps t;
  t.first = __dsub_rn((double)s1, fs1) > 1e-3;
  t.last = __dsub_rn(fs2, (double)s2) > 1e-3;
  t.s0 = t.first ? s1 - 1 : s1;
  t.n = t.first + (s2 - s1) + t.last;
  t.w_first = __double2float_rn(__ddiv_rn(__dsub_rn((double)s1, fs1), cell));
  t.w_mid = __double2float_rn(__ddiv_rn(1.0, cell));
  t.w_last = __double2float_rn(__ddiv_rn(fmin(fmin(__dsub_rn(fs2, (double)s2), 1.0), cell), cell));
  return t;
}

__device__ __forceinline__ float area_weight(const AreaTaps& t, int k) {
  return (k == 0 && t.first) ? t.w_first : (k == t.n - 1 && t.last) ? t.w_last : t.w_mid;
}

// destination pixel (rx, ry) of the INTER_AREA resize of the HWC uint8 image `img` (g.H0 x g.W0 x 3)
__device__ __forceinline__ void resize_area_pixel_u8(const unsigned char* __restrict__ img, const AreaGeom& g, int rx, int ry, int v[3]) {
  if (g.mode == 0) {
    const unsigned char* q = img + ((size_t)ry * g.W0 + rx) * 3;
    v[0] = q[0]; v[1] = q[1]; v[2] = q[2];
  } else if (g.mode == 2) {
    const unsigned char* q0 = img + ((size_t)(2 * ry) * g.W0 + 2 * rx) * 3;
    const unsigned char* q1 = q0 + (size_t)g.W0 * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = (q0[c] + q0[3 + c] + q1[c] + q1[3 + c] + 2) >> 2;
  } else if (g.mode == 3) {                 // resizeAreaFast_Invoker: integer block sum times the float reciprocal of the area
    int s[3] = {0, 0, 0};
    for (int dy = 0; dy < g.ky; ++dy) {
      const unsigned char* q = img + ((size_t)(ry * g.ky + dy) * g.W0 + (size_t)rx * g.kx) * 3;
      for (int dx = 0; dx < g.kx; ++dx)
#pragma unroll
        for (int c = 0; c < 3; ++c) s[c] += q[dx * 3 + c];
    }
    const float inv = __fdiv_rn(1.0f, (float)(g.kx * g.ky));
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = min(255, max(0, __float2int_rn(__fmul_rn((float)s[c], inv))));
  } else {                                  // ResizeArea_Invoker: per y tap a row buffer over the x taps, then sum += beta * buf
    const AreaTaps tx = area_taps(rx, g.scale_x, g.W0), ty = area_taps(ry, g.scale_y, g.H0);
    float sum[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < ty.n; ++j) {
      const unsigned char* row = img + ((size_t)(ty.s0 + j) * g.W0 + tx.s0) * 3;
      float buf[3] = {0.f, 0.f, 0.f};
      for (int k = 0; k < tx.n; ++k) {
        const float a = area_weight(tx, k);
#pragma unroll
        for (int c = 0; c < 3; ++c) buf[c] = __fadd_rn(buf[c], __fmul_rn((float)row[k * 3 + c], a));
      }
      const float beta = area_weight(ty, j);
#pragma unroll
      for (int c = 0; c < 3; ++c) sum[c] = j == 0 ? __fmul_rn(beta, buf[c]) : __fadd_rn(sum[c], __fmul_rn(beta, buf[c]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = min(255, max(0, __float2int_rn(sum[c])));
  }
}

}  // namespace myolo
