// Detection training batches on the device (reference utils/datasets.py:518-593 `LoadImagesAndLabels.__getitem__` with augment=True):
// the image cache resize of `load_image` (:629-643; INTER_LINEAR, and INTER_AREA for the augment=False cache), and ONE fused kernel per batch for the 4-image mosaic (:671-724), the affine
// `random_perspective` warp (:851-893), mixup (:529-532), `augment_hsv` (:646-657), the flips (:571-582) and BGR->RGB / HWC->CHW (:589).
// The host draws the random parameters and transforms the labels (multiyolov5_b200/utils/datasets.py DetAugmenter); this file only moves
// pixels.  The output is S x S (mosaic batches) or H x W (--rect batches, DetRectLoader).  Every step is bit exact with OpenCV 8-bit arithmetic:
//   * cv2.warpAffine INTER_LINEAR / BORDER_CONSTANT 114: 10-bit fixed-point source addresses, 5-bit fractions, 15-bit weights;
//   * the 2s x 2s mosaic canvas is never built: a canvas pixel is the tile covering it, else 114 (also outside the canvas);
//   * cv2.COLOR_BGR2HSV: integer (hsv_shift 12) with rounded division tables;
//   * cv2.COLOR_HSV2BGR: float32 with the (1 - s*h) terms as fused multiply-adds and the result *255 truncated, which is what OpenCV's
//     8-bit path computes (proven over all 180x256x256 inputs by tests/test_augment_host.py against cv2 itself).
// Double precision is written with __dmul_rn / __dadd_rn so that nvcc cannot contract it into fused multiply-adds.
// Parity: tests/test_gpu_augment.py.
#include "kernels.h"
#include "resize.cuh"

namespace myolo {

static_assert(sizeof(myolo_aug_warp) == 200 && sizeof(myolo_aug_item) == 1200, "layout shared with multiyolov5_b200/_lib.py");

__global__ void resize_u8_kernel(const unsigned char* src, ResizeGeom g, unsigned char* dst, int H, int W) {
  const long total = (long)H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    int v[3];
    resize_pixel_u8(src, g, (int)(i % W), (int)(i / W), v);
    dst[i * 3 + 0] = (unsigned char)v[0];
    dst[i * 3 + 1] = (unsigned char)v[1];
    dst[i * 3 + 2] = (unsigned char)v[2];
  }
}

// load_image's augment=False cache resize: cv2.INTER_AREA whenever the image shrinks
__global__ void resize_area_u8_kernel(const unsigned char* __restrict__ src, AreaGeom g, unsigned char* __restrict__ dst, int H, int W) {
  const long total = (long)H * W;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    int v[3];
    resize_area_pixel_u8(src, g, (int)(i % W), (int)(i / W), v);
    dst[i * 3 + 0] = (unsigned char)v[0];
    dst[i * 3 + 1] = (unsigned char)v[1];
    dst[i * 3 + 2] = (unsigned char)v[2];
  }
}

// one of the (up to) four tiles of a warp's virtual canvas
__device__ __forceinline__ void canvas_px(const myolo_aug_warp& w, int cx, int cy, int v[3]) {
  v[0] = v[1] = v[2] = 114;
  for (int t = 0; t < w.n_tiles; ++t) {       // mosaic tiles are disjoint; a later tile would win like the later img4 assignment
    if (cx >= w.rect[t][0] && cy >= w.rect[t][1] && cx < w.rect[t][2] && cy < w.rect[t][3]) {
      const unsigned char* q = w.src[t] + ((size_t)(cy - w.off[t][1]) * w.src_w[t] + (cx - w.off[t][0])) * 3;
      v[0] = __ldg(q); v[1] = __ldg(q + 1); v[2] = __ldg(q + 2);
    }
  }
}

// cv2.warpAffine(canvas, M, (W, H), INTER_LINEAR, BORDER_CONSTANT, 114) at destination pixel (x, y); minv is M inverted as cv2 inverts it
__device__ __forceinline__ void warp_px(const myolo_aug_warp& w, int x, int y, int v[3]) {
  const double* m = w.minv;
  const int adelta = __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)x), 1024.0));
  const int bdelta = __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)x), 1024.0));
  const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), 1024.0)) + 16;
  const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), 1024.0)) + 16;
  const int X = (X0 + adelta) >> 5, Y = (Y0 + bdelta) >> 5;
  const int sx = X >> 5, sy = Y >> 5, fx = X & 31, fy = Y & 31;
  // initInterTab2D's 15-bit weights: float products of multiples of 1/32 are exact, so they round to these integers and their sum is
  // always 2^15 (the table's rounding-error correction never fires)
  const int w00 = (32 - fy) * (32 - fx) * 32, w01 = (32 - fy) * fx * 32, w10 = fy * (32 - fx) * 32, w11 = fy * fx * 32;
  int p00[3], p01[3], p10[3], p11[3];
  canvas_px(w, sx, sy, p00);
  canvas_px(w, sx + 1, sy, p01);
  canvas_px(w, sx, sy + 1, p10);
  canvas_px(w, sx + 1, sy + 1, p11);
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = min(255, max(0, (p00[c] * w00 + p01[c] * w01 + p10[c] * w10 + p11[c] * w11 + (1 << 14)) >> 15));
}

__global__ void __launch_bounds__(256) augment_det_kernel(const myolo_aug_item* __restrict__ items, int B, int H, int W, void* out,
                                                         int out_dtype) {
  __shared__ int sdiv[256], hdiv[256];          // cv2 RGB2HSV_b tables: round((255 << 12) / v), round((180 << 12) / (6 * diff))
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    sdiv[i] = i ? __double2int_rn(__ddiv_rn(255.0 * 4096.0, (double)i)) : 0;
    hdiv[i] = i ? __double2int_rn(__ddiv_rn(180.0 * 4096.0, __dmul_rn(6.0, (double)i))) : 0;
  }
  __syncthreads();
  const long plane = (long)H * W, total = (long)B * plane;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int b = (int)(i / plane);
    const int y = (int)((i % plane) / W), x = (int)(i % W);
    const myolo_aug_item& it = items[b];
    const int ys = it.flipud ? H - 1 - y : y, xs = it.fliplr ? W - 1 - x : x;    // np.flipud / np.fliplr of the augmented image
    int px[3];
    warp_px(it.warp[0], xs, ys, px);
    if (it.n_warps == 2) {                       // mixup: (img * r + img2 * (1 - r)).astype(np.uint8) in float64
      int px2[3];
      warp_px(it.warp[1], xs, ys, px2);
#pragma unroll
      for (int c = 0; c < 3; ++c) px[c] = (int)__dadd_rn(__dmul_rn((double)px[c], it.mix_r), __dmul_rn((double)px2[c], it.mix_q));
    }
    // ---- augment_hsv: BGR -> HSV (integer), LUTs, HSV -> BGR
    const int bb = px[0], gg = px[1], rr = px[2];
    const int vmax = max(bb, max(gg, rr)), vmin = min(bb, min(gg, rr)), diff = vmax - vmin;
    const int vr = vmax == rr ? -1 : 0, vg = vmax == gg ? -1 : 0;
    const int sat = (diff * sdiv[vmax] + (1 << 11)) >> 12;
    int hue = (vr & (gg - bb)) + (~vr & ((vg & (bb - rr + 2 * diff)) + ((~vg) & (rr - gg + 4 * diff))));
    hue = (hue * hdiv[diff] + (1 << 11)) >> 12;
    hue += hue < 0 ? 180 : 0;
    const float hf = (float)it.lut[0][hue];
    const float sf = __fmul_rn((float)it.lut[1][sat], 1.0f / 255.0f);
    const float vf = __fmul_rn((float)it.lut[2][vmax], 1.0f / 255.0f);
    const float hx = __fmul_rn(hf, 6.0f / 180.0f);
    const float sector_f = floorf(hx);
    const float fr = __fsub_rn(hx, sector_f);
    const float tab1 = __fmul_rn(vf, __fsub_rn(1.0f, sf));
    const float tab2 = __fmul_rn(vf, __fmaf_rn(-sf, fr, 1.0f));
    const float tab3 = __fmul_rn(vf, __fmaf_rn(-sf, __fsub_rn(1.0f, fr), 1.0f));
    int sector = (int)sector_f;
    sector = sector < 0 || sector > 5 ? 0 : sector;
    // sector -> (b, g, r) entries of the table (v, tab1, tab2, tab3): {1,3,0} {1,0,2} {3,0,1} {0,2,1} {0,1,3} {2,1,0}, 2 bits each, 6 bits per sector
    const unsigned long long code = 0x0Dull | (0x21ull << 6) | (0x13ull << 12) | (0x18ull << 18) | (0x34ull << 24) | (0x06ull << 30);
    const unsigned sel = (unsigned)(code >> (6 * sector)) & 63u;
    int bgr[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) {                // selects instead of an indexed array: keeps the table in registers
      const unsigned k = (sel >> (2 * c)) & 3u;
      const float t = k == 0 ? vf : k == 1 ? tab1 : k == 2 ? tab2 : tab3;
      bgr[c] = (int)__fmul_rn(t, 255.0f);      // truncation, as cv2's 8-bit path
    }
    // ---- BGR -> RGB, HWC -> CHW
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const int val = bgr[2 - c];
      const size_t o = ((size_t)b * 3 + c) * plane + (size_t)y * W + x;
      if (out_dtype == MYOLO_U8) reinterpret_cast<unsigned char*>(out)[o] = (unsigned char)val;
      // imgs.float() / 255 on a CUDA tensor (reference train.py:342): ATen multiplies by the fp32 reciprocal of a scalar divisor
      else if (out_dtype == MYOLO_F16) reinterpret_cast<__half*>(out)[o] = __float2half_rn(__fmul_rn((float)val, 1.0f / 255.0f));
      else reinterpret_cast<float*>(out)[o] = __fmul_rn((float)val, 1.0f / 255.0f);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// --multi-scale (reference train.py:354-359): F.interpolate(imgs, size=ns, mode='bilinear', align_corners=False) of the det batch, bit
// exact with ATen's CUDA kernel (UpSampleBilinear2d.cu upsample_bilinear2d_out_frame).  The host passes ATen's scales, float(in) / out.
// ATen's expressions with nvcc's contractions as they appear in the sm_90 SASS of the kernel torch launches:
//   src  = fma(dst + 0.5, scale, -0.5), clamped at 0 (area_pixel_compute_source_index);  i1 = trunc(src);  l1 = src - i1;  l0 = 1 - l1
//   val  = fma(h0l, fma(w0l, a, w1l * b), h1l * fma(w0l, c, w1l * d))      a..d: taps (h1,w1) (h1,w1+w1p) (h1+h1p,w1) (h1+h1p,w1+w1p)
// uint8 taps are first converted as `imgs.float() / 255.0` converts them on the device (train.py:342): v * fp32(1/255).
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float bilinear_tap(const T* p);
template <>
__device__ __forceinline__ float bilinear_tap<unsigned char>(const unsigned char* p) { return __fmul_rn((float)__ldg(p), 1.0f / 255.0f); }
template <>
__device__ __forceinline__ float bilinear_tap<__half>(const __half* p) { return __half2float(__ldg(p)); }
template <>
__device__ __forceinline__ float bilinear_tap<float>(const float* p) { return __ldg(p); }

__device__ __forceinline__ void bilinear_source(int d, int n_in, float scale, int* i0, int* i1, float* l0, float* l1) {
  float src = __fmaf_rn(__fadd_rn((float)d, 0.5f), scale, -0.5f);
  src = src < 0.f ? 0.f : src;
  const int i = (int)src;
  *i0 = i;
  *i1 = i + (i < n_in - 1 ? 1 : 0);
  *l1 = __fsub_rn(src, (float)i);
  *l0 = __fsub_rn(1.0f, *l1);
}

// one thread per output pixel of one (image, channel) plane; grid (x tiles, rows, planes)
template <typename Ts, typename Td>
__global__ void __launch_bounds__(128) resize_bilinear_kernel(const Ts* __restrict__ src, int planes, int H, int W, Td* __restrict__ dst,
                                                              int Ho, int Wo, float rh, float rw) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= Wo) return;
  const bool same = H == Ho && W == Wo;      // scale 1: the conversion alone
  int h0 = y, h1 = y, w0 = x, w1 = x;
  float h0l = 1.f, h1l = 0.f, w0l = 1.f, w1l = 0.f;
  if (!same) {
    bilinear_source(y, H, rh, &h0, &h1, &h0l, &h1l);
    bilinear_source(x, W, rw, &w0, &w1, &w0l, &w1l);
  }
  for (int p = blockIdx.z; p < planes; p += gridDim.z) {
    const Ts* s = src + (size_t)p * H * W;
    float val;
    if (same) {
      val = bilinear_tap(s + (size_t)y * W + x);
    } else {
      const float a = bilinear_tap(s + (size_t)h0 * W + w0), b = bilinear_tap(s + (size_t)h0 * W + w1);
      const float c = bilinear_tap(s + (size_t)h1 * W + w0), d = bilinear_tap(s + (size_t)h1 * W + w1);
      const float top = __fmaf_rn(w0l, a, __fmul_rn(w1l, b));
      const float bot = __fmaf_rn(w0l, c, __fmul_rn(w1l, d));
      val = __fmaf_rn(h0l, top, __fmul_rn(h1l, bot));
    }
    const size_t o = ((size_t)p * Ho + y) * Wo + x;
    if constexpr (sizeof(Td) == 2) dst[o] = __float2half_rn(val);
    else dst[o] = val;
  }
}

template <typename Ts>
static void launch_resize_bilinear_from(const Ts* src, int planes, int H, int W, void* dst, int dst_dtype, int Ho, int Wo, float rh, float rw,
                                        cudaStream_t s) {
  const dim3 grid((Wo + 127) / 128, Ho, std::min(planes, 65535));
  if (dst_dtype == MYOLO_F16) resize_bilinear_kernel<Ts, __half><<<grid, 128, 0, s>>>(src, planes, H, W, (__half*)dst, Ho, Wo, rh, rw);
  else resize_bilinear_kernel<Ts, float><<<grid, 128, 0, s>>>(src, planes, H, W, (float*)dst, Ho, Wo, rh, rw);
}

// ------------------------------------------------------------------------------------------------
// scale_img (reference utils/torch_utils.py:248-258) of test-time augmentation, optionally of x.flip(3): F.interpolate to (Ho, Wo) as
// resize_bilinear_kernel computes it, then F.pad on the right and bottom to (Hp, Wp) with `pad` (already rounded to the dtype by the
// host; Hp < Ho or Wp < Wo crops, as F.pad's negative padding does).  flip reads source column W-1-w: the interpolation of the mirrored
// image.  One thread per output pixel of one plane; grid (x tiles, rows, planes).
// ------------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) scale_img_kernel(const T* __restrict__ src, int planes, int H, int W, T* __restrict__ dst, int Ho,
                                                        int Wo, int Hp, int Wp, float rh, float rw, int flip, float pad) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= Wp) return;
  const bool inside = y < Ho && x < Wo;
  const bool same = H == Ho && W == Wo;
  int h0 = y, h1 = y, w0 = x, w1 = x;
  float h0l = 1.f, h1l = 0.f, w0l = 1.f, w1l = 0.f;
  if (inside && !same) {
    bilinear_source(y, H, rh, &h0, &h1, &h0l, &h1l);
    bilinear_source(x, W, rw, &w0, &w1, &w0l, &w1l);
  }
  if (flip) { w0 = W - 1 - w0; w1 = W - 1 - w1; }
  for (int p = blockIdx.z; p < planes; p += gridDim.z) {
    const T* s = src + (size_t)p * H * W;
    float val = pad;
    if (inside && same) {
      val = bilinear_tap(s + (size_t)h0 * W + w0);
    } else if (inside) {
      const float a = bilinear_tap(s + (size_t)h0 * W + w0), b = bilinear_tap(s + (size_t)h0 * W + w1);
      const float c = bilinear_tap(s + (size_t)h1 * W + w0), d = bilinear_tap(s + (size_t)h1 * W + w1);
      const float top = __fmaf_rn(w0l, a, __fmul_rn(w1l, b));
      const float bot = __fmaf_rn(w0l, c, __fmul_rn(w1l, d));
      val = __fmaf_rn(h0l, top, __fmul_rn(h1l, bot));
    }
    const size_t o = ((size_t)p * Hp + y) * Wp + x;
    if constexpr (sizeof(T) == 2) dst[o] = __float2half_rn(val);
    else dst[o] = val;
  }
}

// ------------------------------------------------------------------------------------------------
// --quad (reference utils/datasets.py:602-625 LoadImagesAndLabels.collate_fn4): quad q of the output is either the 2x2 tile of items
// 4q (top left), 4q+1 (bottom left), 4q+2 (top right), 4q+3 (bottom right), or
//   F.interpolate(img[4q].float()[None], scale_factor=2., mode='bilinear', align_corners=False)[0].type(uint8)
// computed in integers.  With scale 1/2 the source coordinate of output row Y is Y/2 - 1/4 clamped at 0, so an even row 2r takes rows
// (r-1, r) with weights (1/4, 3/4) and an odd row 2r+1 rows (r, r+1) with (3/4, 1/4); row 0 and a last odd row take one row with weight 1,
// which is the same sum with the missing row clamped to its neighbour.  Columns likewise.  Every partial result torch forms is a multiple
// of 1/16 in [0, 256) and so exact in fp32, whatever its order of evaluation (tests/test_quad_host.py proves it), and the truncating
// uint8 cast is floor(sum / 16) of the integer sum with weights {1, 3} x {1, 3}.
// ------------------------------------------------------------------------------------------------
struct QuadFlags {                   // a __grid_constant__ parameter: indexed in place, not copied to local memory
  unsigned w[MYOLO_QUAD_MAX / 32];   // bit q: quad q is the 2x2 tile, else the x2 upsample of its first item
};

__device__ __forceinline__ bool quad_is_tile(const QuadFlags& f, int q) { return (f.w[q >> 5] >> (q & 31)) & 1u; }

// the float outputs are imgs.float() / 255 on the device (reference train.py:342), as augment_det_kernel writes them
__device__ __forceinline__ float quad_unit(int v) { return __fmul_rn((float)v, 1.0f / 255.0f); }

// 8 consecutive output pixels [X0, X0 + 8) of row Y in one (quad, channel) plane; W % 8 == 0, so X0 is 8-aligned, a tile never straddles
// an 8-pixel group, and every load and store below is naturally aligned
template <int OUT>
__global__ void __launch_bounds__(256) collate_quad_vec_kernel(const unsigned char* __restrict__ imgs, int H, int W,
                                                               const __grid_constant__ QuadFlags flags, void* __restrict__ out) {
  const int Wo = 2 * W, Ho = 2 * H, groups = Wo >> 3;
  const long gid = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (gid >= (long)Ho * groups) return;
  const int plane = blockIdx.y, q = plane / 3, c = plane - 3 * q;
  const int Y = (int)(gid / groups), X0 = (int)(gid - (long)Y * groups) << 3;
  const size_t HW = (size_t)H * W;
  int v[8];
  if (quad_is_tile(flags, q)) {
    const int item = 4 * q + (Y >= H ? 1 : 0) + (X0 >= W ? 2 : 0);     // cat over H (i, i+1) then over W ((i, i+1), (i+2, i+3))
    const int y = Y >= H ? Y - H : Y, x = X0 >= W ? X0 - W : X0;
    const uint2 p = __ldg(reinterpret_cast<const uint2*>(imgs + ((size_t)item * 3 + c) * HW + (size_t)y * W + x));
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = (p.x >> (8 * j)) & 255u;
      v[4 + j] = (p.y >> (8 * j)) & 255u;
    }
  } else {
    const unsigned char* src = imgs + ((size_t)(4 * q) * 3 + c) * HW;
    const int r = Y >> 1;
    const int ya = (Y & 1) ? r : max(r - 1, 0), yb = (Y & 1) ? min(r + 1, H - 1) : r;   // weights (3, 1) for odd rows, (1, 3) for even
    const int wa = (Y & 1) ? 3 : 1, wb = 4 - wa;
    const int k = X0 >> 1;                                                               // source columns k-1 .. k+4, clamped
    int h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = 0;
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      const unsigned char* row = src + (size_t)(t ? yb : ya) * W;
      const int wy = t ? wb : wa;
      const unsigned mid = __ldg(reinterpret_cast<const unsigned*>(row + k));
      int a[6];
      a[0] = __ldg(row + max(k - 1, 0));
#pragma unroll
      for (int j = 0; j < 4; ++j) a[1 + j] = (mid >> (8 * j)) & 255u;
      a[5] = __ldg(row + min(k + 4, W - 1));
#pragma unroll
      for (int m = 0; m < 4; ++m) {                       // output columns 2(k+m) and 2(k+m)+1
        h[2 * m] += wy * (a[m] + 3 * a[m + 1]);
        h[2 * m + 1] += wy * (3 * a[m + 1] + a[m + 2]);
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = h[j] >> 4;
  }
  const size_t o = ((size_t)plane * Ho + Y) * Wo + X0;
  if (OUT == MYOLO_U8) {
    uint2 p;
    p.x = v[0] | (v[1] << 8) | (v[2] << 16) | ((unsigned)v[3] << 24);
    p.y = v[4] | (v[5] << 8) | (v[6] << 16) | ((unsigned)v[7] << 24);
    *reinterpret_cast<uint2*>(reinterpret_cast<unsigned char*>(out) + o) = p;
  } else if (OUT == MYOLO_F16) {
    __align__(16) __half hv[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) hv[j] = __float2half_rn(quad_unit(v[j]));
    *reinterpret_cast<uint4*>(reinterpret_cast<__half*>(out) + o) = *reinterpret_cast<const uint4*>(hv);
  } else {
    float4* d = reinterpret_cast<float4*>(reinterpret_cast<float*>(out) + o);
    d[0] = make_float4(quad_unit(v[0]), quad_unit(v[1]), quad_unit(v[2]), quad_unit(v[3]));
    d[1] = make_float4(quad_unit(v[4]), quad_unit(v[5]), quad_unit(v[6]), quad_unit(v[7]));
  }
}

// any W or alignment: one output pixel per thread, the same arithmetic with byte loads
__global__ void __launch_bounds__(256) collate_quad_kernel(const unsigned char* __restrict__ imgs, int H, int W,
                                                           const __grid_constant__ QuadFlags flags, void* __restrict__ out, int out_dtype) {
  const int Wo = 2 * W, Ho = 2 * H;
  const long gid = blockIdx.x * (long)blockDim.x + threadIdx.x;
  if (gid >= (long)Ho * Wo) return;
  const int plane = blockIdx.y, q = plane / 3, c = plane - 3 * q;
  const int Y = (int)(gid / Wo), X = (int)(gid - (long)Y * Wo);
  const size_t HW = (size_t)H * W;
  int v;
  if (quad_is_tile(flags, q)) {
    const int item = 4 * q + (Y >= H ? 1 : 0) + (X >= W ? 2 : 0);
    v = __ldg(imgs + ((size_t)item * 3 + c) * HW + (size_t)(Y >= H ? Y - H : Y) * W + (X >= W ? X - W : X));
  } else {
    const unsigned char* src = imgs + ((size_t)(4 * q) * 3 + c) * HW;
    const int r = Y >> 1, k = X >> 1;
    const int ya = (Y & 1) ? r : max(r - 1, 0), yb = (Y & 1) ? min(r + 1, H - 1) : r, wya = (Y & 1) ? 3 : 1;
    const int xa = (X & 1) ? k : max(k - 1, 0), xb = (X & 1) ? min(k + 1, W - 1) : k, wxa = (X & 1) ? 3 : 1;
    const unsigned char* ra = src + (size_t)ya * W;
    const unsigned char* rb = src + (size_t)yb * W;
    const int top = wxa * __ldg(ra + xa) + (4 - wxa) * __ldg(ra + xb);
    const int bot = wxa * __ldg(rb + xa) + (4 - wxa) * __ldg(rb + xb);
    v = (wya * top + (4 - wya) * bot) >> 4;
  }
  const size_t o = ((size_t)plane * Ho + Y) * Wo + X;
  if (out_dtype == MYOLO_U8) reinterpret_cast<unsigned char*>(out)[o] = (unsigned char)v;
  else if (out_dtype == MYOLO_F16) reinterpret_cast<__half*>(out)[o] = __float2half_rn(quad_unit(v));
  else reinterpret_cast<float*>(out)[o] = quad_unit(v);
}

}  // namespace myolo

using namespace myolo;

extern "C" int myolo_resize_u8(const uint8_t* src, int H0, int W0, uint8_t* dst, int H, int W, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && dst && H0 > 0 && W0 > 0 && H > 0 && W > 0, "resize_u8: bad geometry (src %dx%d dst %dx%d)", W0, H0, W, H);
  const long total = (long)H * W;
  resize_u8_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(src, resize_geom(H0, W0, H, W), dst, H, W);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_resize_area_u8(const uint8_t* src, int H0, int W0, uint8_t* dst, int H, int W, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && dst && H0 > 0 && W0 > 0 && H > 0 && W > 0, "resize_area_u8: bad geometry (src %dx%d dst %dx%d)", W0, H0, W, H);
  MYOLO_REQUIRE(H <= H0 && W <= W0, "resize_area_u8: down-scaling only (src %dx%d dst %dx%d)", W0, H0, W, H);
  const long total = (long)H * W;
  resize_area_u8_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(src, area_geom(H0, W0, H, W), dst, H, W);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_augment_det_hw(const myolo_aug_item* items, int B, int H, int W, void* out, int out_dtype, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(items && out && B > 0 && H > 0 && W > 0, "augment_det: bad arguments (B %d H %d W %d)", B, H, W);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "augment_det: output dtype");
  const long total = (long)B * H * W;
  augment_det_kernel<<<(int)std::min<long>(132L * 16, (total + 255) / 256), 256, 0, s>>>(items, B, H, W, out, out_dtype);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_resize_bilinear(const void* src, int src_dtype, int B, int C, int H, int W, void* dst, int dst_dtype, int Ho, int Wo,
                                     void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && dst && B > 0 && C > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Ho <= 65535,
                "resize_bilinear: bad geometry (B %d C %d src %dx%d dst %dx%d)", B, C, H, W, Ho, Wo);
  MYOLO_REQUIRE(src_dtype == MYOLO_U8 || src_dtype == MYOLO_F16 || src_dtype == MYOLO_F32, "resize_bilinear: source dtype %d", src_dtype);
  MYOLO_REQUIRE(dst_dtype == MYOLO_F16 || dst_dtype == MYOLO_F32, "resize_bilinear: output dtype %d", dst_dtype);
  MYOLO_REQUIRE((long)B * C <= (1L << 31) - 1, "resize_bilinear: too many planes");
  const int planes = B * C;
  // area_pixel_compute_scale with no scale factor given: static_cast<float>(input_size) / output_size, in fp32 on the host
  const float rh = (float)H / (float)Ho, rw = (float)W / (float)Wo;
  if (src_dtype == MYOLO_U8) launch_resize_bilinear_from((const unsigned char*)src, planes, H, W, dst, dst_dtype, Ho, Wo, rh, rw, s);
  else if (src_dtype == MYOLO_F16) launch_resize_bilinear_from((const __half*)src, planes, H, W, dst, dst_dtype, Ho, Wo, rh, rw, s);
  else launch_resize_bilinear_from((const float*)src, planes, H, W, dst, dst_dtype, Ho, Wo, rh, rw, s);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_scale_img(const void* src, int dtype, int B, int C, int H, int W, void* dst, int Ho, int Wo, int Hp, int Wp, int flip_lr,
                               float pad, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(src && dst && B > 0 && C > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && Hp > 0 && Wp > 0 && Hp <= 65535,
                "scale_img: bad geometry (B %d C %d src %dx%d resized %dx%d padded %dx%d)", B, C, H, W, Ho, Wo, Hp, Wp);
  MYOLO_REQUIRE(dtype == MYOLO_F16 || dtype == MYOLO_F32, "scale_img: dtype %d (fp16 or fp32 only)", dtype);
  MYOLO_REQUIRE((long)B * C <= (1L << 31) - 1, "scale_img: too many planes");
  const int planes = B * C;
  const float rh = (float)H / (float)Ho, rw = (float)W / (float)Wo;     // area_pixel_compute_scale, as in myolo_resize_bilinear
  const dim3 grid((Wp + 127) / 128, Hp, std::min(planes, 65535));
  if (dtype == MYOLO_F16)
    scale_img_kernel<__half><<<grid, 128, 0, s>>>((const __half*)src, planes, H, W, (__half*)dst, Ho, Wo, Hp, Wp, rh, rw, flip_lr != 0, pad);
  else
    scale_img_kernel<float><<<grid, 128, 0, s>>>((const float*)src, planes, H, W, (float*)dst, Ho, Wo, Hp, Wp, rh, rw, flip_lr != 0, pad);
  MYOLO_LAUNCH_CHECK();
  return 0;
}

extern "C" int myolo_collate_quad(const uint8_t* imgs, int B, int H, int W, const uint8_t* tile, void* out, int out_dtype, void* stream) {
  if (int rc = check_device(nullptr)) return rc;
  const cudaStream_t s = (cudaStream_t)stream;
  MYOLO_REQUIRE(imgs && out && tile && B >= 4 && H > 0 && W > 0, "collate_quad: bad arguments (B %d H %d W %d)", B, H, W);
  MYOLO_REQUIRE(B / 4 <= MYOLO_QUAD_MAX, "collate_quad: %d quads, at most %d", B / 4, MYOLO_QUAD_MAX);
  MYOLO_REQUIRE((long)H * W <= (1L << 28), "collate_quad: %dx%d images are too large", H, W);
  MYOLO_REQUIRE(out_dtype == MYOLO_U8 || out_dtype == MYOLO_F16 || out_dtype == MYOLO_F32, "collate_quad: output dtype %d", out_dtype);
  const int n = B / 4;
  QuadFlags f = {};
  for (int q = 0; q < n; ++q)
    if (tile[q]) f.w[q >> 5] |= 1u << (q & 31);
  const long Ho = 2L * H, Wo = 2L * W;
  if (W % 8 == 0 && ((uintptr_t)imgs & 7) == 0 && ((uintptr_t)out & 15) == 0) {
    const dim3 grid((unsigned)((Ho * (Wo / 8) + 255) / 256), 3 * n);
    if (out_dtype == MYOLO_U8) collate_quad_vec_kernel<MYOLO_U8><<<grid, 256, 0, s>>>(imgs, H, W, f, out);
    else if (out_dtype == MYOLO_F16) collate_quad_vec_kernel<MYOLO_F16><<<grid, 256, 0, s>>>(imgs, H, W, f, out);
    else collate_quad_vec_kernel<MYOLO_F32><<<grid, 256, 0, s>>>(imgs, H, W, f, out);
  } else {
    const dim3 grid((unsigned)((Ho * Wo + 255) / 256), 3 * n);
    collate_quad_kernel<<<grid, 256, 0, s>>>(imgs, H, W, f, out, out_dtype);
  }
  MYOLO_LAUNCH_CHECK();
  return 0;
}
