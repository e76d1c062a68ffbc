// Host-side description of one fused conv op (Conv / Bottleneck.cv2 / bare Conv2d+BN+SiLU / Detect.m[i] / classifier).
#pragma once
#include "common.cuh"

namespace myolo {

// division by a runtime constant as multiply-high + shift (the tile decode runs once per tile in EVERY epilogue warp: three hardware
// divisions there cost ~800 clk per tile under the epilogue's issue pressure - measured with the clock64 timeline)
struct FastDiv {
  unsigned mul, shr;
};
static inline FastDiv make_fastdiv(unsigned d) {     // exact for 0 <= n < 2^31, d >= 1
  unsigned l = 0;
  while ((1ull << l) < d) ++l;
  FastDiv f;
  f.mul = (unsigned)((((1ull << l) - d) << 32) / d + 1);
  f.shr = l;
  return f;
}

struct ConvTcParams {
  int B, Ho, Wo;
  int tw, th;            // output tile = tw x th pixels, tw*th == 128 (two wgmma M = 64 halves)
  int log2_tw;
  int tiles_x, tiles_y;  // per image
  int n_tiles_n, total_tiles;
  int BN;                // wgmma N (multiple of 16, <= 128)
  int Co;                // real output channels
  int kc;                // channels per K chunk: 16 / 32 / 64  (swizzle 32B / 64B / 128B)
  int cblocks;           // Ci_pad / kc
  int taps;              // k*k
  int n_chunks, n_kstages;
  int tap_map[9], tap_dx[9], tap_dy[9];
  int act;
  int num_stages;
  int a_stage_bytes, b_stage_bytes;
  int resident;          // 1: the CTA's whole weight slice stays in shared memory (one slot per K chunk), loaded by its first tile
  int b_bytes;           // shared memory of the weight region: resident slots or num_stages ring stages
  int bias_bytes;        // shared memory of the bias vector: n_tiles_n * BN floats, 128-byte aligned
  int strip;             // 1: 3x3 stride 1, one A box {kc, tw + 2 dil, th} per filter row and channel block feeds the row's three taps
  int strip_w;           // tw + 2 dil: pixels per strip row
  int strip_box_bytes, strip_sub_bytes;   // bytes of one strip box / its 1024-aligned slot in the stage
  int dil;
  int out_mode;          // 0: fp16 NHWC slice, 1: fp32 NHWC slice
  int out_c, out_ctot;   // channels of the output slice (fp32: min(out_c, Co) are stored) / channel pitch of its buffer
  const float* bias;
  const __half* residual;  // nullable; base of the residual slice (image 0, pixel 0, channel 0 of the slice)
  int res_ctot;
  __half* out_f16;
  float* out_f32;
  FastDiv fd_ntn, fd_tpi, fd_tx;   // n_tiles_n, tiles_x * tiles_y, tiles_x
};

struct ConvOp {
  TensorView in, out, res;
  bool has_res = false;
  int k = 1, stride = 1, dil = 1, act = MYOLO_ACT_SILU;
  const __half* w = nullptr;  // packed [Co_pad][k*k*Ci_pad]
  const float* bias = nullptr;
  int Ci_pad = 0, Co_pad = 0, Co = 0;
  bool use_tc = false;
  bool reuse = true;          // false: streamed weights, one ring stage per K step (the reference layout of the standalone entry's path 3)
  // tensor-core path state (built once at plan creation)
  CUtensorMap tmA[4], tmB;
  ConvTcParams p;
  int grid = 0, smem = 0;
  int ctas_per_sm = 1;        // resident CTAs per SM the launch is sized for (conv_tc_prepare)
};

// decides whether the tensor-core (wgmma) path can run this op (the output and residual views must already be resolved: their
// base pointers are checked for 16-byte alignment)
bool conv_tc_eligible(const ConvOp& op);
// builds tensor maps / params; requires op.in/out/res/w/bias device pointers to be final
int conv_tc_prepare(ConvOp& op, int num_sms);
int conv_tc_launch(const ConvOp& op, cudaStream_t stream);
int conv_simt_launch(const ConvOp& op, cudaStream_t stream);
int conv_simt_launch_group(const ConvOp* const* ops, int n, cudaStream_t stream);   // <= 4 small convs of one input type in one launch

// weight packing: fp32 [Co][Ci][k][k] (+BN) -> fp16 [Co_pad][k*k][Ci_pad], bias fp32 [Co_pad]
// one job of the grouped weight pack (conv_simt.cu pack_group_kernel)
static constexpr int kPackChunk = 2048;
struct PackJob {
  const float* w;
  const float *gamma, *beta, *mean, *var, *bias;
  __half* wp;
  float* bp;
  int co, ci, k;
  int n_pad, c_pad;      // kind 0: (co_pad, ci_pad);  kind 1: (ci_pad_out, co_pad_in)
  float eps;
  int kind;
  int chunk0;            // first chunk (= block) of this job
};
int pack_group_launch(const PackJob* d_jobs, int n_jobs, int total_chunks, cudaStream_t stream);
int pack_conv_weights(const float* w, int co, int ci, int k, const float* gamma, const float* beta, const float* mean,
                      const float* var, float eps, const float* bias, __half* wp, float* bp, int co_pad, int ci_pad,
                      cudaStream_t stream);

}  // namespace myolo
