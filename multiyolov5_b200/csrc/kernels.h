// Launchers of the HBM-bound (non-GEMM) kernels of the path.  All take resolved TensorViews (NHWC) unless noted.
#pragma once
#include "common.cuh"

namespace myolo {

// Focus.forward slicing + NCHW->NHWC + cast (reference models/common.py:549-550, detect.py:135-137)
int launch_input_focus(const void* x, int x_dtype, int B, int H, int W, const TensorView& out, cudaStream_t s);
int launch_upsample_nearest2x(const TensorView& in, const TensorView& out, cudaStream_t s);
// SPP: out slices 1..3 = maxpool 5/9/13 of slice 0 (views share one buffer); reference models/common.py:170-174
int launch_spp_pool(const TensorView& in, const TensorView& out5, int n_cascade, cudaStream_t s);
int launch_bilinear_nhwc(const TensorView& in, const TensorView& out, cudaStream_t s);
int launch_bilinear_nhwc_group(const TensorView* in, const TensorView* out, int n, cudaStream_t s);
int launch_region_combine_group(const TensorView& atoms, int atoms_nx, const int* const* d_bins, const int* nbins, const TensorView* out, int n,
                                cudaStream_t s);
int launch_region_sum(const TensorView& in, const int* d_ybounds, int ny, const int* d_xbounds, int nx, const TensorView& out,
                      cudaStream_t s);
int launch_region_combine(const TensorView& atoms, int atoms_nx, const int* d_bins, int nbins, const TensorView& out,
                          cudaStream_t s);
int launch_channel_scale(const TensorView& feat, const TensorView& att, cudaStream_t s);
int launch_add(const TensorView& a, const TensorView& b, const TensorView& out, cudaStream_t s);
int launch_broadcast(const TensorView& in, const TensorView& out, cudaStream_t s);
// Detect.forward (reference models/yolo.py:211-225): in = fp32 NHWC conv output (channel = a*no + o).  Test-time augmentation
// (models/yolo.py:274-289): z's four box columns are multiplied by z_inv_scale, and z_flip_w > 0 replaces x by z_flip_w - x
int launch_detect_decode(const TensorView& in, int na, int no, float stride, const float* d_anchors /*na*2 px*/, float* raw,
                         float* z, int z_row_offset, int z_rows_total, cudaStream_t s, float z_inv_scale = 1.0f, int z_flip_w = 0);
// final bilinear(align_corners) of the seg head: in = fp32 NHWC low-res logits; seg NCHW (fp32/fp16, nullable); argmax nullable
int launch_seg_upsample(const TensorView& in, int n_cls, int H, int W, void* seg, int seg_dtype, int64_t* argmax,
                        cudaStream_t s);
// the ensemble's seg (myolo_seg_ensemble): ins[0..K) = the members' fp32 NHWC low-res logits (same extents)
int launch_seg_ensemble(const TensorView* ins, int K, int n_cls, int H, int W, void* seg, int seg_dtype, int64_t* argmax, cudaStream_t s);
int launch_read_view(const TensorView& v, float* dst_nchw, cudaStream_t s);

}  // namespace myolo
