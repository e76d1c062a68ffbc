// Training-mode kernels of the path (SURVEY.md section 8 row a13): batch-statistics BatchNorm forward, and the backward of every op kind
// the *_city_seg PSP graph uses.  Activations and activation gradients are NHWC fp16 (loss scaling is the caller's, like the reference's
// amp.GradScaler, train.py:265,371); parameter gradients are accumulated in fp32 straight into the caller's .grad tensors.
#pragma once
#include "common.cuh"
#include "conv.h"

namespace myolo {

struct BnParams {           // device pointers owned by the caller (nn.BatchNorm2d tensors), fp32
  float* gamma = nullptr;
  float* beta = nullptr;
  float* running_mean = nullptr;
  float* running_var = nullptr;
  float* d_gamma = nullptr;  // .grad (accumulated), nullable
  float* d_beta = nullptr;
  float momentum = 0.03f, eps = 1e-3f;
  int C = 0;
  bool set = false;
};

// ---- forward ----
// per-channel mean / inverse std over (B,H,W) of u (fp16 NHWC view) -> stats[0..C) = mean, stats[C..2C) = invstd; updates running stats
int launch_bn_stats(const TensorView& u, const BnParams& bn, float* stats, float* scratch, cudaStream_t s, bool defer_running = false);
struct RunningJob {         // one BN layer of a deferred running-statistics update (batch_stats = [mean | biased variance] of npix values)
  float* running_mean;
  float* running_var;
  const float* batch_stats;
  int C;
  long npix;
  float momentum;
};
int launch_bn_apply_running(const RunningJob* d_jobs, int n_jobs, cudaStream_t s);
// synchronised BatchNorm (torch.nn.SyncBatchNorm).  A rank's record is kBnRecHead + 2*C floats: {count as int32 bits, 0, 0, 0, mean[C],
// biased var[C]}; records of all ranks lie back to back (what ncclAllGather of one record per rank produces).
constexpr int kBnRecHead = 4;
// the record of u (C % 8 == 0, C <= 2048) into rec; scratch as launch_bn_stats'.  Finalises nothing.
int launch_bn_stats_record(const TensorView& u, const BnParams& bn, float* rec, float* scratch, cudaStream_t s);
// global mean / invstd -> stats, running statistics with the global count, *inv_n = 1 / N (device) from n_rec gathered records
int launch_bn_sync_combine(const float* recs, int n_rec, const BnParams& bn, float* stats, float* inv_n, cudaStream_t s);
// sums[0..n) += sums[g*n .. g*n+n) for g = 1 .. n_groups-1, in order
int launch_bn_sync_sum(float* sums, int n_groups, int n, cudaStream_t s);
// y = act(gamma*(u-mean)*invstd + beta) (+ residual)
int launch_bn_act_fwd(const TensorView& u, const TensorView* res, const TensorView& y, const BnParams& bn, const float* stats, int act,
                      cudaStream_t s);
// elementwise activation on tiny fp32 maps (FFM attention): y = act(x)
int launch_act_fwd(const TensorView& x, const TensorView& y, int act, cudaStream_t s);
// out = f * (1 + a)   (out-of-place FFM scale for training)
int launch_channel_scale_oop(const TensorView& f, const TensorView& a, const TensorView& out, cudaStream_t s);

int launch_dropout(const TensorView& x, const TensorView& y, float p, unsigned long long seed, const unsigned long long* step, unsigned salt,
                   int accumulate, cudaStream_t s);
int launch_bump_step(unsigned long long* step, cudaStream_t s);

// ---- backward ----
// dz = dy*act'(z), z = gamma*xhat+beta; du = gamma*invstd*(dz - mean(dz) - xhat*mean(dz*xhat)); dgamma += sum(dz*xhat); dbeta += sum(dz)
// d_res (nullable) += dy.  `scratch` holds 2*C floats.  Synchronised BN: synced_sums = {sum dz, sum dz*xhat} over all ranks (2*C
// floats) and inv_n = 1 / N (device) replace the local reduce and 1 / npix.
int launch_bn_act_bwd(const TensorView& u, const TensorView& dy, const TensorView& du, const TensorView* d_res, const BnParams& bn,
                      const float* stats, int act, float* scratch, cudaStream_t s, const float* synced_sums = nullptr,
                      const float* inv_n = nullptr);
// the local {sum dz, sum dz*xhat} of a synchronised BN layer into sums_out (2*C floats); adds them to d_beta / d_gamma as well
int launch_bn_bwd_sums(const TensorView& u, const TensorView& dy, const BnParams& bn, const float* stats, int act, float* scratch,
                       float* sums_out, cudaStream_t s);
int launch_act_bwd(const TensorView& x, const TensorView& dy, const TensorView& dx, int act, cudaStream_t s);
// df += dout*(1+a);  da[b,c] += sum_p dout*f
int launch_channel_scale_bwd(const TensorView& f, const TensorView& a, const TensorView& dout, const TensorView& df, const TensorView& da,
                             cudaStream_t s);
int launch_grad_add(const TensorView& src, const TensorView& dst, cudaStream_t s);                    // dst += src
int launch_broadcast_bwd(const TensorView& dout, const TensorView& din, cudaStream_t s);             // din(1x1) += spatial sum
int launch_nearest2x_bwd(const TensorView& dout, const TensorView& din, cudaStream_t s);             // din += 2x2 sums
size_t bilinear_bwd_scratch_bytes(const TensorView& dout, const TensorView& din);
int launch_bilinear_bwd(const TensorView& dout, const TensorView& din, float* scratch, cudaStream_t s);  // din += adjoint(align_corners)
int launch_spp_bwd(const TensorView& x, const TensorView& dout3, const TensorView& dx, float* scratch_f32, cudaStream_t s);
int launch_region_bwd(const TensorView& datoms_or_bins, const TensorView& dx, const int* d_yb, int ny, const int* d_xb, int nx,
                      cudaStream_t s);                                                                // dx[p] += datoms[atom(p)]
int launch_region_combine_bwd(const TensorView& dbins, const TensorView& datoms, int atoms_nx, const int* d_bins, int nbins,
                              cudaStream_t s);                                                        // datoms += dbin/count
// seg head: d(low-res logits fp32 NHWC) += adjoint of the final bilinear applied to dseg (B,C,H,W) fp32
int launch_seg_upsample_bwd(const float* dseg, int n_cls, int H, int W, const TensorView& dlo, cudaStream_t s);
// fused CE(ignore_index) of the bilinear-upsampled low-res logits: seeds d(low-res logits) += factor * (*scale_dev) * d(mean CE)/d(lo)
// and writes the mean CE to loss_out (device, nullable); scratch16 = 16 bytes of device scratch.  With ohem_ws (ohem_scratch_bytes(B*H*W)
// bytes) the loss is OhemCELoss's instead: the pixels a device-side selection takes (loss > thresh_t, or the n_valid // 16 largest)
size_t seg_ce_scratch_bytes(int B, int H, int W, int n_cls);
size_t ohem_scratch_bytes(long n_pixels);
int launch_seg_ce_fused(const TensorView& lo, int n_cls, const long long* labels, int H, int W, int ignore_index, const TensorView& dlo,
                        float factor, const float* scale_dev, void* scratch16, float* gbuf, float* loss_out, cudaStream_t s,
                        void* ohem_ws = nullptr, float thresh_t = 0.f);
// the same fused pass with the class-weighted CE / focal loss (weights: n_cls device floats, nullable; gamma = 0 is the weighted CE) in
// place of the mean CE, reduction 'mean'; wf_ws: seg_wf_scratch_bytes(B*H*W) bytes (the loss's sums and coefficients, 8 bytes per pixel)
size_t seg_wf_scratch_bytes(long n_pixels);
int launch_seg_wf_fused(const TensorView& lo, int n_cls, const long long* labels, int H, int W, int ignore_index, const TensorView& dlo,
                        float factor, const float* scale_dev, float* gbuf, void* wf_ws, const float* weights, float gamma, float* loss_out,
                        cudaStream_t s);
// Detect: d(conv out fp32 NHWC)[b,y,x,a*no+o] = draw[b,a,y,x,o]
int launch_detect_raw_bwd(const float* draw, int na, int no, const TensorView& dconv, cudaStream_t s);
int launch_cast_f32_to_f16(const TensorView& src, const TensorView& dst, cudaStream_t s);
int launch_cast_f16_to_f32_acc(const TensorView& src, const TensorView& dst, cudaStream_t s);        // dst(f32) += src(f16)
// conv parameter gradients: dW[co][ci][ky][kx] += sum_p dY[p][co] * X[p*stride + tap][ci];  dbias[co] += sum_p dY[p][co]
int launch_conv_wgrad(const TensorView& x, const TensorView& dy, int k, int stride, int dil, float* dW, int co, int ci, float* dbias,
                      cudaStream_t s);
int launch_bias_grad(const TensorView& dy, float* dbias, int co, cudaStream_t s);                     // dbias[co] += sum_p dy (fp32 or fp16 view)
// wgmma weight gradient (wgrad_tc.cu): dw_packed is a zeroed fp32 [co][k*k][ci] accumulation buffer owned by the caller
bool conv_wgrad_tc_eligible(const TensorView& x, const TensorView& dy, int k, int stride, int dil, int co, int ci);
size_t conv_wgrad_packed_bytes(const float* dW, int co, int ci, int k);   // 0: accumulates straight into dW
// tiling (nullable): {pixels per step Kc, N, row slabs, rows per slab, rows in all}
int launch_conv_wgrad_tc(const TensorView& x, const TensorView& dy, int k, int stride, int dil, float* dW, float* dw_packed, int co, int ci,
                         int num_sms, cudaStream_t s, int32_t* tiling = nullptr);
// tiny maps / fp32 tensors: generic backward straight from the fp32 master weights (dx nullable: += ; dW += ; dbias += )
int launch_conv_small_bwd(const TensorView& x, const TensorView& dy, const TensorView* dx, const float* w, float* dW, float* dbias, int co,
                          int ci, int k, int stride, int dil, cudaStream_t s);
// dgrad weights: fp32 [Co][Ci][k][k] -> fp16 [Ci_pad][k*k (flipped)][Co_pad]  (a conv of dY with these weights is the data gradient)
int pack_dgrad_weights(const float* w, int co, int ci, int k, __half* wp, float* zero_bias, int ci_pad_out, int co_pad_in, cudaStream_t s);
// stride-2 data gradient helper: dst (2H x 2W, zero) gets src at even positions (transposed conv == stride-1 conv on the stuffed map)
int launch_zero_stuff2(const TensorView& src, const TensorView& dst, cudaStream_t s);

}  // namespace myolo
