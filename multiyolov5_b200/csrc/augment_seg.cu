// Segmentation training batches on the device (reference SegmentationDataset.py:118-151 `_sync_transform`, :182-189 `_class_to_index`,
// and the loader functions' ColorJitter + ToTensor, :458-531), and the testval items (:81-94).  Two launches per batch:
//   1. seg_resample_kernel: Pillow's bilinear Image.resize of the (optionally mirrored) source, evaluated only over the crop window (the
//      resized image is never stored), the right/bottom pad (image 0, mask 255), the NEAREST mask resize and the mask -> label LUT.  It also
//      accumulates, per item, the sum of L of the image as it enters adjust_contrast (the jitter ops before contrast are per pixel).
//   2. seg_jitter_kernel: the item's jitter ops in its randperm order, then ToTensor (v / 255) and HWC -> CHW.
// The host (multiyolov5_b200/utils/datasets.py SegAugmenter) draws the parameters and builds the per-item resampling tables in double
// as Pillow's precompute_coeffs / normalize_coeffs_8bpc and ImagingScaleAffine compute them.  Every step is bit exact with Pillow:
//   * resample: 22-bit fixed point, horizontal rows rounded and clipped to uint8 before the vertical pass (an unchanged axis gets a one-tap
//     identity table, which reproduces Pillow's skipped pass);
//   * Image.blend: in1 + alpha * (in2 - in1) in float, truncated for 0 <= alpha <= 1 and clipped otherwise;
//   * convert("L") integer; convert("HSV") and back with Pillow's float / double mix;
//   * contrast's mean int(sum / n + 0.5) in double, as ImageStat computes it.
// Float and double arithmetic is written with __f*_rn / __d*_rn so that nvcc cannot contract it into fused multiply-adds; the restatement
// it follows (restate_seg.py) is checked against Pillow over the whole input domain of each operation.  Parity:
// tests/test_gpu_seg_augment.py.
#include "kernels.h"

namespace myolo {

static_assert(sizeof(myolo_seg_item) == 1120, "layout shared with multiyolov5_b200/_lib.py");

__device__ __forceinline__ int clip8(int v) { return min(255, max(0, v)); }

// Image.blend(in1, in2, alpha) of one channel
__device__ __forceinline__ int blend_u8(int in1, int in2, float a) {
  const float t = __fadd_rn((float)in1, __fmul_rn(a, (float)(in2 - in1)));
  if (a >= 0.0f && a <= 1.0f) return (int)t;
  return t <= 0.0f ? 0 : t >= 255.0f ? 255 : (int)t;
}

__device__ __forceinline__ int luma(const int c[3]) { return (c[0] * 19595 + c[1] * 38470 + c[2] * 7471 + 0x8000) >> 16; }

// adjust_hue: convert("HSV") (rgb2hsv_row), H += shift in uint8, HSV -> RGB (hsv2rgb)
__device__ __forceinline__ void hue_u8(int c[3], int shift) {
  const int r = c[0], g = c[1], b = c[2];
  const int mx = max(r, max(g, b)), mn = min(r, min(g, b));
  int uh = 0, us = 0;
  if (mx != mn) {
    const float cr = (float)(mx - mn);
    const float s = __fdiv_rn(cr, (float)mx);
    const float rc = __fdiv_rn((float)(mx - r), cr), gc = __fdiv_rn((float)(mx - g), cr), bc = __fdiv_rn((float)(mx - b), cr);
    float h;
    if (r == mx) h = __fsub_rn(bc, gc);
    else if (g == mx) h = __double2float_rn(__dsub_rn(__dadd_rn(2.0, (double)rc), (double)bc));
    else h = __double2float_rn(__dsub_rn(__dadd_rn(4.0, (double)gc), (double)rc));
    h = __double2float_rn(fmod(__dadd_rn(__ddiv_rn((double)h, 6.0), 1.0), 1.0));
    uh = clip8((int)__dmul_rn((double)h, 255.0));
    us = clip8((int)__dmul_rn((double)s, 255.0));
  }
  const int hh = (uh + shift) & 255, s = us, v = mx;
  if (s == 0) {
    c[0] = c[1] = c[2] = v;
    return;
  }
  const double hd = __ddiv_rn(__dmul_rn((double)hh, 6.0), 255.0);
  const int i = (int)floor(hd);
  const float f = __double2float_rn(__dsub_rn(hd, (double)i));
  const float fs = __fmul_rn(f, (float)s);
  const double vd = (double)v;
  const int p = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, __ddiv_rn((double)s, 255.0)))));
  const int q = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, __ddiv_rn((double)fs, 255.0)))));
  const int t = clip8((int)round(__dmul_rn(vd, __dsub_rn(1.0, __ddiv_rn((double)__fsub_rn((float)s, fs), 255.0)))));
  switch (i % 6) {
    case 0: c[0] = v; c[1] = t; c[2] = p; break;
    case 1: c[0] = q; c[1] = v; c[2] = p; break;
    case 2: c[0] = p; c[1] = v; c[2] = t; break;
    case 3: c[0] = p; c[1] = q; c[2] = v; break;
    case 4: c[0] = t; c[1] = p; c[2] = v; break;
    default: c[0] = v; c[1] = p; c[2] = q; break;
  }
}

// the item's jitter ops in order; stops before contrast when `upto_contrast` (the image whose L mean contrast needs)
__device__ __forceinline__ void jitter(const myolo_seg_item& it, int c[3], int mean, bool upto_contrast) {
#pragma unroll 1
  for (int k = 0; k < 4; ++k) {
    const int op = it.order[k];
    if (op < 0 || (upto_contrast && op == 1)) return;
    if (op == 0) {
#pragma unroll
      for (int j = 0; j < 3; ++j) c[j] = blend_u8(0, c[j], it.factor[0]);
    } else if (op == 1) {
#pragma unroll
      for (int j = 0; j < 3; ++j) c[j] = blend_u8(mean, c[j], it.factor[1]);
    } else if (op == 2) {
      const int l = luma(c);
#pragma unroll
      for (int j = 0; j < 3; ++j) c[j] = blend_u8(l, c[j], it.factor[2]);
    } else {
      hue_u8(c, it.hue_shift);
    }
  }
}

__device__ __forceinline__ bool has_contrast(const myolo_seg_item& it) {
  return it.order[0] == 1 || it.order[1] == 1 || it.order[2] == 1 || it.order[3] == 1;
}

// crop pixel (X, Y) of the bilinear resize: tables hold {first source index, taps, coefficients} per crop column / row (taps 0 = pad)
__device__ __forceinline__ void resample_px(const myolo_seg_item& it, const int* __restrict__ tables, int X, int Y, int c[3]) {
  const int* ce = tables + it.col + X * (it.kx + 2);
  const int* re = tables + it.row + Y * (it.ky + 2);
  const int cs = ce[0], cn = ce[1], rs = re[0], rn = re[1];
  c[0] = c[1] = c[2] = 0;
  if (cn == 0 || rn == 0) return;
  int acc[3] = {1 << 21, 1 << 21, 1 << 21};
  for (int j = 0; j < rn; ++j) {
    const unsigned char* row = it.img + (size_t)(rs + j) * it.W0 * 3;
    int h[3] = {1 << 21, 1 << 21, 1 << 21};
    for (int i = 0; i < cn; ++i) {
      const int sx = it.flip ? it.W0 - 1 - (cs + i) : cs + i;
      const unsigned char* p = row + (size_t)sx * 3;
      const int k = ce[2 + i];
      h[0] += __ldg(p) * k;
      h[1] += __ldg(p + 1) * k;
      h[2] += __ldg(p + 2) * k;
    }
    const int kv = re[2 + j];
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) acc[ch] += clip8(h[ch] >> 22) * kv;
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) c[ch] = clip8(acc[ch] >> 22);
}

__global__ void __launch_bounds__(256) seg_resample_kernel(myolo_seg_item* __restrict__ items, int h, int w, int mh, int mw,
                                                           const int* __restrict__ tables, unsigned char* __restrict__ scratch,
                                                           long long* __restrict__ out_mask) {
  const int b = blockIdx.y;
  const myolo_seg_item& it = items[b];
  const bool contrast = has_contrast(it);
  const long n_img = (long)h * w, n_mask = (long)mh * mw, n = max(n_img, n_mask);
  unsigned long long lsum = 0;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < n; i += (long)gridDim.x * blockDim.x) {
    if (i < n_img) {
      const int Y = (int)(i / w), X = (int)(i % w);
      int c[3];
      resample_px(it, tables, X, Y, c);
      unsigned char* o = scratch + ((size_t)b * n_img + i) * 3;
      o[0] = (unsigned char)c[0];
      o[1] = (unsigned char)c[1];
      o[2] = (unsigned char)c[2];
      if (contrast) {
        jitter(it, c, 0, true);
        lsum += (unsigned long long)luma(c);
      }
    }
    if (i < n_mask) {
      const int Y = (int)(i / mw), X = (int)(i % mw);
      const int mx = tables[it.mcol + X], my = tables[it.mrow + Y];
      const int v = (mx < 0 || my < 0) ? 255 : __ldg(it.mask + (size_t)my * it.W0 + (it.flip ? it.W0 - 1 - mx : mx));
      out_mask[(size_t)b * n_mask + i] = it.lut[v];
    }
  }
  if (!contrast) return;
  __shared__ unsigned long long part[8];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lsum += __shfl_down_sync(0xffffffffu, lsum, o);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = lsum;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long s = 0;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) s += part[k];
    atomicAdd(reinterpret_cast<unsigned long long*>(&items[b].lsum), s);
  }
}

__global__ void __launch_bounds__(256) seg_jitter_kernel(const myolo_seg_item* __restrict__ items, int h, int w,
                                                         const unsigned char* __restrict__ scratch, void* out, int out_dtype) {
  const int b = blockIdx.y;
  const myolo_seg_item& it = items[b];
  const long plane = (long)h * w;
  // ImageEnhance.Contrast: int(ImageStat mean + 0.5), the mean a double division of the exact integer sum
  const int mean = (int)__dadd_rn(__ddiv_rn((double)it.lsum, (double)plane), 0.5);
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < plane; i += (long)gridDim.x * blockDim.x) {
    const unsigned char* p = scratch + ((size_t)b * plane + i) * 3;
    int c[3] = {p[0], p[1], p[2]};
    jitter(it, c, mean, false);
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const size_t o = ((size_t)b * 3 + ch) * plane + i;
      // ToTensor: uint8 -> float32, then a true division by 255 (not a multiplication by its reciprocal)
      const float f = __fdiv_rn((float)c[ch], 255.0f);
      if (out_dtype == MYOLO_U8) reinterpret_cast<unsigned char*>(out)[o] = (unsigned char)c[ch];
      else if (out_dtype == MYOLO_F16) reinterpret_cast<__half*>(out)[o] = __float2half_rn(f);
      else reinterpret_cast<float*>(out)[o] = f;
    }
  }
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_augment_seg(myolo_seg_item* items, int B, int h, int w, int mh, int mw, const int32_t* tables, uint8_t* scratch,
                                 void* out, int out_dtype, int64_t* out_mask, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(items && tables && scratch && out && out_mask && B > 0 && h > 0 && w > 0 && mh > 0 && mw > 0 && B <= 65535,
                "augment_seg: bad arguments (B %d image %dx%d mask %dx%d)", B, w, h, mw, mh);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "augment_seg: output dtype");
  const long n = std::max((long)h * w, (long)mh * mw);
  const int per_item = (int)std::max<long>(1, std::min<long>((n + 255) / 256, (132L * 16 + B - 1) / B));
  seg_resample_kernel<<<dim3(per_item, B), 256, 0, s>>>(items, h, w, mh, mw, tables, scratch, reinterpret_cast<long long*>(out_mask));
  MYOLO_LAUNCH_CHECK();
  const int per_item2 = (int)std::max<long>(1, std::min<long>(((long)h * w + 255) / 256, (132L * 16 + B - 1) / B));
  seg_jitter_kernel<<<dim3(per_item2, B), 256, 0, s>>>(items, h, w, scratch, out, out_dtype);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
