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
int launch_read_view(const TensorView& v, float* dst_nchw, cudaStream_t s);

// pre-process (preprocess.cu): letterbox resize + border + channel swap / layout / dtype conversion of uint8 HWC frames
int launch_letterbox(const unsigned char* src, int B, int H0, int W0, int rw, int rh, int top, int left, int H, int W, const int* pad3,
                     void* dst, int out_dtype, int chw, int swap_rb, cudaStream_t s);
int launch_letterbox_items(const unsigned char* src, const myolo_letterbox_item* items, int B, int H, int W, void* dst, int out_dtype,
                           cudaStream_t s);

// detection training batches (augment.cu): image cache resize and the fused mosaic / warp / mixup / HSV / flip kernel
int launch_resize_u8(const unsigned char* src, int H0, int W0, unsigned char* dst, int H, int W, cudaStream_t s);
int launch_resize_area_u8(const unsigned char* src, int H0, int W0, unsigned char* dst, int H, int W, cudaStream_t s);
int launch_augment_det(const myolo_aug_item* items, int B, int H, int W, void* out, int out_dtype, cudaStream_t s);
int launch_resize_bilinear(const void* src, int src_dtype, int B, int C, int H, int W, void* dst, int dst_dtype, int Ho, int Wo, cudaStream_t s);
int launch_scale_img(const void* src, int dtype, int B, int C, int H, int W, void* dst, int Ho, int Wo, int Hp, int Wp, int flip_lr, float pad,
                     cudaStream_t s);
int launch_collate_quad(const unsigned char* imgs, int B, int H, int W, const unsigned char* tile, void* out, int out_dtype, cudaStream_t s);

// segmentation training batches (augment_seg.cu): crop-window resample + pad + mask LUT, then the ColorJitter / ToTensor kernel
int launch_augment_seg(myolo_seg_item* items, int B, int h, int w, int mh, int mw, const int* tables, unsigned char* scratch, void* out,
                       int out_dtype, long long* out_mask, cudaStream_t s);

// detection validation statistics (metrics.cu): per-batch matching into the stats store, ap_per_class over the whole store
int launch_confusion(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets, int H, int W,
                     const float* geom, int nc, float conf_thres, float iou_thres, int require_rows, unsigned long long* matrix, int32_t* err,
                     cudaStream_t s);
int launch_det_match(const float* dets, const int32_t* counts, int B, int max_det, const float* targets, int n_targets, int H, int W,
                     const float* geom, const float* iouv, int img_base, uint16_t* st_correct, float* st_conf, uint8_t* st_cls,
                     int32_t* st_rows, unsigned long long* tcount, int32_t* err, cudaStream_t s);
int64_t det_ap_workspace_bytes(int n_images, int max_det, int ncol);
int launch_det_ap(const uint16_t* correct, const float* conf, const uint8_t* cls, const int32_t* rows, int n_images, int max_det, int ncol,
                  const unsigned long long* tcount, const double* px, const double* x101, double* out_ap, double* out_p, double* out_r,
                  int32_t* out_info, void* workspace, int64_t workspace_bytes, cudaStream_t s);

// seg output consumers (consumers.cu)
int launch_lut_blend(const void* idx, int idx_dtype, long n, const unsigned char* lut, int n_entries, int ch, int reverse, unsigned char* out,
                     const unsigned char* im, float alpha, float beta, unsigned char* blend, const unsigned char* lut2, int ch2,
                     unsigned char* out2, cudaStream_t s);
int launch_detect_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, int nc, float* xywhn, int32_t* class_counts,
                        cudaStream_t s);
int launch_scale_boxes(float* rows, const int32_t* counts, int B, int max_det, const float* geom, float* xywh, float* xyxyn, float* xywhn,
                       cudaStream_t s);
int launch_seg_hist(const void* pred, int pred_dtype, const long long* target, long n, int n_cls, unsigned long long* counters, cudaStream_t s);

// autoanchor (autoanchor.cu): the ratio metric and the cooperative genetic evolution
int64_t anchor_metric_workspace_bytes();
int launch_anchor_metric(const void* wh, int wh_dtype, long n, const void* k, int k_dtype, int na, double thr, myolo_anchor_stats* out,
                         void* workspace, cudaStream_t s);
int anchor_evolve_workspace_bytes(long n, int64_t* bytes);
int launch_anchor_evolve(const float* wh, long n, const double* k0, int na, const double* v, int gen, float thr, double* k_out,
                         float* f_out, float* fg_out, int* accepted_out, void* workspace, int64_t workspace_bytes, cudaStream_t s);

// scipy's k-means (kmeans.cu): one CTA per restart
int64_t kmeans_workspace_bytes(long n, int restarts);
int launch_kmeans(const double* obs, long n, const int64_t* init_idx, int k, int restarts, double thresh, int max_iter, double* books,
                  int32_t* book_k, double* dists, int32_t* iters, int32_t* best, int32_t* status, void* ws, int64_t ws_bytes,
                  cudaStream_t s);

// --image-weights (image_weights.cu): class weights, image weights, the weighted draw
int launch_class_weights(const float* cls, long long n_labels, int nc, unsigned long long* counts, double* weights, int32_t* status,
                         cudaStream_t s);
int launch_image_weights(const float* cls, const int64_t* offsets, long long n, const double* cw, int nc, double* iw, int32_t* status,
                         cudaStream_t s);
int launch_weighted_draw(const double* w, const double* u, long long n, double* cum, double* total, int32_t* idx, int32_t* status,
                         cudaStream_t s);

}  // namespace myolo
