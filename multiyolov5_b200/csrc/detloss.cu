// Detection loss of the training step, forward AND backward, in four launches (reference utils/loss.py:115-217 `ComputeLoss.__call__` +
// `build_targets`, and torch.autograd through them): CIoU box loss on the matched cells, BCE objectness against the (detached) IoU of the last
// matching candidate of every cell, BCE class loss.  The torch formulation of the same arithmetic (multiyolov5_b200/utils/loss.py, ~760 tiny
// kernels replayed as a CUDA graph) cost milliseconds of the step; this is four launches.
//
//   candidates of level l: (offset o in {0, +x, +y, -x, -y}) x (anchor a) x (target t), exactly the reference's candidate order
//       cand = (o * na + a) * nt + t                                  (utils/loss.py:198-207: targets are repeated per anchor, then per offset)
//   valid   = anchor ratio test  max(r, 1/r) < anchor_t   AND   (o == 0 or the neighbouring cell on that side is the nearer one)
//   cell    = (b, a, clamp(gj), clamp(gi)),  tbox = (gxy - clamped cell, gwh)     (the reference clamps IN PLACE on a view of gij, :211-212)
//   lbox_l  = mean over valid of (1 - CIoU(pbox, tbox));   pbox = (2 sigma(xy) - 0.5, (2 sigma(wh))^2 * anchor)
//   tobj    = (1 - gr) + gr * clamp(IoU, 0) of the LAST valid candidate of the cell (what the reference's CPU index_put_ leaves)
//   lcls_l  = mean over valid x classes of BCE(logit, cp / cn);   lobj_l = mean over all cells of BCE(obj logit, tobj)
//   loss    = bs * (box * sum lbox_l + obj * sum balance_l lobj_l + cls * sum lcls_l)
// Restrictions (the reference's defaults, data/hyp.scratch.yaml): fl_gamma = 0, cls_pw = obj_pw = 1, no autobalance; the Python wrapper falls
// back to the torch formulation otherwise.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace myolo {

struct DetLossParams {
  const float* p[3];
  float* dp[3];
  int ny[3], nx[3];
  float anchors[3][2 * MYOLO_DET_LOSS_NA_MAX];   // [level][a*2 + {w,h}] in grid units (kernel parameter: 240 bytes at na = 10)
  float balance[3];
  int nl, B, na, no, nc, nt;
  const float* targets;     // (nt, 6): image, class, x, y, w, h (normalised)
  float hyp_box, hyp_obj, hyp_cls, anchor_t, gr, cp, cn;
  float mult;               // bs * world * detgain (host constant)
  const float* scale;       // device loss scale (nullable)
  int* winner[3];           // per cell: index of the last valid candidate, -1 = none
  float* tobj[3];           // per cell objectness target
  int* nvalid;              // [3]
  float* sums;              // [3][3]: lbox, lobj, lcls per level (unnormalised parts are normalised where they are added)
  float* items;             // out: lbox, lobj, lcls, loss (detached, like ComputeLoss's loss_items)
};

struct Cand { bool valid; int b, a, gj, gi, cls; float tx, ty, tw, th; };

__device__ __forceinline__ Cand decode_cand(const DetLossParams& P, int l, int cand) {
  Cand c;
  const int t = cand % P.nt;
  const int a = (cand / P.nt) % P.na;
  const int o = cand / (P.nt * P.na);
  const float* T = P.targets + (size_t)t * 6;
  const float nx = (float)P.nx[l], ny = (float)P.ny[l];
  const float gx = T[2] * nx, gy = T[3] * ny, gw = T[4] * nx, gh = T[5] * ny;
  const float aw = P.anchors[l][a * 2], ah = P.anchors[l][a * 2 + 1];
  const float rw = gw / aw, rh = gh / ah;
  const bool match = fmaxf(fmaxf(rw, 1.0f / rw), fmaxf(rh, 1.0f / rh)) < P.anchor_t;
  bool sel = true;
  float ox = 0.f, oy = 0.f;
  if (o == 1) { sel = (fmodf(gx, 1.0f) < 0.5f) && (gx > 1.0f); ox = 0.5f; }
  else if (o == 2) { sel = (fmodf(gy, 1.0f) < 0.5f) && (gy > 1.0f); oy = 0.5f; }
  else if (o == 3) { const float q = nx - gx; sel = (fmodf(q, 1.0f) < 0.5f) && (q > 1.0f); ox = -0.5f; }
  else if (o == 4) { const float q = ny - gy; sel = (fmodf(q, 1.0f) < 0.5f) && (q > 1.0f); oy = -0.5f; }
  c.valid = match && sel;
  c.a = a;
  c.b = (int)T[0];
  c.cls = (int)T[1];
  const int gi = (int)(gx - ox), gj = (int)(gy - oy);                 // .long(): truncation toward zero
  c.gi = min(max(gi, 0), P.nx[l] - 1);
  c.gj = min(max(gj, 0), P.ny[l] - 1);
  c.tx = gx - (float)c.gi;
  c.ty = gy - (float)c.gj;
  c.tw = gw;
  c.th = gh;
  return c;
}

__device__ __forceinline__ float warp_sum_f(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + __expf(-x)); }
// F.softplus (beta 1, threshold 20)
__device__ __forceinline__ float softplusf_(float x) { return x > 20.0f ? x : log1pf(__expf(x)); }

// phase A: count the valid candidates of each level and find the last valid candidate of every cell
__global__ void det_assign_kernel(DetLossParams P) {
  const int l = blockIdx.y;
  const int ncand = 5 * P.na * P.nt;
  for (int cand = blockIdx.x * blockDim.x + threadIdx.x; cand < ncand; cand += gridDim.x * blockDim.x) {
    const Cand c = decode_cand(P, l, cand);
    if (!c.valid) continue;
    atomicAdd(P.nvalid + l, 1);
    const int cell = ((c.b * P.na + c.a) * P.ny[l] + c.gj) * P.nx[l] + c.gi;
    atomicMax(P.winner[l] + cell, cand);
  }
}

// phase B: box + class loss and their gradients on the matched cells; objectness targets
__global__ void det_match_kernel(DetLossParams P) {
  const int l = blockIdx.y;
  const int ncand = 5 * P.na * P.nt;
  const float eps = 1e-7f;
  const float n = fmaxf((float)P.nvalid[l], 1.0f);
  const float gmul = P.mult * (P.scale ? *P.scale : 1.0f);
  float lbox = 0.f, lcls = 0.f;
  for (int cand = blockIdx.x * blockDim.x + threadIdx.x; cand < ncand; cand += gridDim.x * blockDim.x) {
    const Cand c = decode_cand(P, l, cand);
    if (!c.valid) continue;
    const int cell = ((c.b * P.na + c.a) * P.ny[l] + c.gj) * P.nx[l] + c.gi;
    const float* ps = P.p[l] + (size_t)cell * P.no;
    float* dps = P.dp[l] + (size_t)cell * P.no;
    const float aw = P.anchors[l][c.a * 2], ah = P.anchors[l][c.a * 2 + 1];
    const float s0 = sigmoidf_(ps[0]), s1 = sigmoidf_(ps[1]), s2 = sigmoidf_(ps[2]), s3 = sigmoidf_(ps[3]);
    const float px = 2.0f * s0 - 0.5f, py = 2.0f * s1 - 0.5f;
    const float pw = 4.0f * s2 * s2 * aw, ph = 4.0f * s3 * s3 * ah;
    // ---- CIoU forward (reference utils/general.py:343-380, x1y1x2y2=False) ----
    const float px1 = px - pw * 0.5f, px2 = px + pw * 0.5f, py1 = py - ph * 0.5f, py2 = py + ph * 0.5f;
    const float tx1 = c.tx - c.tw * 0.5f, tx2 = c.tx + c.tw * 0.5f, ty1 = c.ty - c.th * 0.5f, ty2 = c.ty + c.th * 0.5f;
    const float iw_raw = fminf(px2, tx2) - fmaxf(px1, tx1), ih_raw = fminf(py2, ty2) - fmaxf(py1, ty1);
    const float iw = fmaxf(iw_raw, 0.f), ih = fmaxf(ih_raw, 0.f);
    const float inter = iw * ih;
    const float w1 = px2 - px1, h1 = py2 - py1 + eps, w2 = tx2 - tx1, h2 = ty2 - ty1 + eps;
    const float uni = w1 * h1 + w2 * h2 - inter + eps;
    const float iou = inter / uni;
    const float cw = fmaxf(px2, tx2) - fminf(px1, tx1), ch = fmaxf(py2, ty2) - fminf(py1, ty1);
    const float c2 = cw * cw + ch * ch + eps;
    const float sx = tx1 + tx2 - px1 - px2, sy = ty1 + ty2 - py1 - py2;
    const float rho2 = (sx * sx + sy * sy) * 0.25f;
    const float k4pi2 = 0.40528473456935109f;          // 4 / pi^2
    const float r1 = w1 / h1;
    const float dv = atanf(w2 / h2) - atanf(r1);
    const float v = k4pi2 * dv * dv;
    const float alpha = v / (v - iou + (1.0f + eps));   // no_grad in the reference
    const float ciou = iou - (rho2 / c2 + v * alpha);
    lbox += (1.0f - ciou) / n;
    // ---- CIoU backward: g_X = d ciou / d X ----
    const float g_rho2 = -1.0f / c2, g_c2 = rho2 / (c2 * c2), g_v = -alpha;
    float g_inter = 1.0f / uni;
    const float g_uni = -inter / (uni * uni);
    float g_w1 = g_uni * h1, g_h1 = g_uni * w1;
    g_inter -= g_uni;
    const float g_iw = g_inter * ih, g_ih = g_inter * iw;
    const float g_iwr = iw_raw >= 0.f ? g_iw : 0.f, g_ihr = ih_raw >= 0.f ? g_ih : 0.f;
    float g_px1 = 0.f, g_px2 = 0.f, g_py1 = 0.f, g_py2 = 0.f;
    if (px2 <= tx2) g_px2 += g_iwr;
    if (px1 >= tx1) g_px1 -= g_iwr;
    if (py2 <= ty2) g_py2 += g_ihr;
    if (py1 >= ty1) g_py1 -= g_ihr;
    const float g_cw = g_c2 * 2.0f * cw, g_ch = g_c2 * 2.0f * ch;
    if (px2 >= tx2) g_px2 += g_cw;
    if (px1 <= tx1) g_px1 -= g_cw;
    if (py2 >= ty2) g_py2 += g_ch;
    if (py1 <= ty1) g_py1 -= g_ch;
    g_px1 += g_rho2 * (-0.5f * sx); g_px2 += g_rho2 * (-0.5f * sx);
    g_py1 += g_rho2 * (-0.5f * sy); g_py2 += g_rho2 * (-0.5f * sy);
    const float g_at1 = -(g_v * 2.0f * k4pi2 * dv);
    const float g_r1 = g_at1 / (1.0f + r1 * r1);
    g_w1 += g_r1 / h1;
    g_h1 -= g_r1 * w1 / (h1 * h1);
    g_px2 += g_w1; g_px1 -= g_w1; g_py2 += g_h1; g_py1 -= g_h1;
    const float g_px = g_px1 + g_px2, g_py = g_py1 + g_py2, g_pw = 0.5f * (g_px2 - g_px1), g_ph = 0.5f * (g_py2 - g_py1);
    // d loss / d logits: loss contains hyp_box * (1 - ciou) / n  (times bs * ... = gmul)
    const float kb = -P.hyp_box * gmul / n;
    atomicAdd(dps + 0, kb * g_px * 2.0f * s0 * (1.0f - s0));
    atomicAdd(dps + 1, kb * g_py * 2.0f * s1 * (1.0f - s1));
    atomicAdd(dps + 2, kb * g_pw * 8.0f * s2 * s2 * (1.0f - s2) * aw);
    atomicAdd(dps + 3, kb * g_ph * 8.0f * s3 * s3 * (1.0f - s3) * ah);
    // ---- class BCE ----
    if (P.nc > 1) {
      const float kc = P.hyp_cls * gmul / (n * (float)P.nc);
      for (int k = 0; k < P.nc; ++k) {
        const float x = ps[5 + k];
        const float t = (k == c.cls) ? P.cp : P.cn;
        lcls += ((1.0f - t) * x + softplusf_(-x)) / (n * (float)P.nc);
        atomicAdd(dps + 5 + k, kc * (sigmoidf_(x) - t));
      }
    }
    if (P.winner[l][cell] == cand) P.tobj[l][cell] = (1.0f - P.gr) + P.gr * fmaxf(ciou, 0.f);   // `iou` of utils/loss.py:138-150 IS the CIoU
  }
  lbox = warp_sum_f(lbox);
  lcls = warp_sum_f(lcls);
  if ((threadIdx.x & 31) == 0) {
    if (lbox != 0.f) atomicAdd(P.sums + l * 3 + 0, lbox);
    if (lcls != 0.f) atomicAdd(P.sums + l * 3 + 2, lcls);
  }
}

// phase C: objectness BCE over every cell of every level, gradient written in place (channel 4 belongs to this kernel alone)
__global__ void det_obj_kernel(DetLossParams P) {
  const int l = blockIdx.y;
  const int ncell = P.B * P.na * P.ny[l] * P.nx[l];
  const float gmul = P.mult * (P.scale ? *P.scale : 1.0f);
  const float kg = P.hyp_obj * P.balance[l] * gmul / (float)ncell;
  float lobj = 0.f;
  for (int cell = blockIdx.x * blockDim.x + threadIdx.x; cell < ncell; cell += gridDim.x * blockDim.x) {
    const float x = P.p[l][(size_t)cell * P.no + 4];
    const float t = P.tobj[l][cell];
    lobj += (1.0f - t) * x + softplusf_(-x);
    P.dp[l][(size_t)cell * P.no + 4] = kg * (sigmoidf_(x) - t);
  }
  lobj = warp_sum_f(lobj);
  if ((threadIdx.x & 31) == 0 && lobj != 0.f) atomicAdd(P.sums + l * 3 + 1, lobj / (float)ncell);
}

__global__ void det_items_kernel(DetLossParams P) {
  float lbox = 0.f, lobj = 0.f, lcls = 0.f;
  for (int l = 0; l < P.nl; ++l) {
    lbox += P.sums[l * 3 + 0];
    lobj += P.sums[l * 3 + 1] * P.balance[l];
    lcls += P.sums[l * 3 + 2];
  }
  lbox *= P.hyp_box; lobj *= P.hyp_obj; lcls *= P.hyp_cls;
  P.items[0] = lbox; P.items[1] = lobj; P.items[2] = lcls; P.items[3] = lbox + lobj + lcls;
}

}  // namespace myolo

using namespace myolo;

extern "C" int64_t myolo_det_loss_workspace_bytes(int B, int na, int nl, const int32_t* ny, const int32_t* nx) {
  int64_t cells = 0;
  for (int l = 0; l < nl; ++l) cells += (int64_t)B * na * ny[l] * nx[l];
  return cells * 8 + 256;
}

extern "C" int myolo_det_loss(const float* const* p, float* const* dp, const float* targets, int nt, int B, int na, int no, int nl,
                              const int32_t* ny, const int32_t* nx, const float* anchors_grid, const float* balance, float hyp_box,
                              float hyp_obj, float hyp_cls, float anchor_t, float gr, float cp, float cn, float mult, const float* scale_dev,
                              float* items_out, void* workspace, int64_t workspace_bytes, void* stream) {
  MYOLO_REQUIRE(p && dp && items_out && workspace && nl >= 1 && nl <= 3 && na >= 1 && na <= MYOLO_DET_LOSS_NA_MAX && no >= 6 && B > 0 && nt >= 0,
                "det_loss: bad arguments");
  MYOLO_REQUIRE(nt == 0 || targets, "det_loss: targets missing");
  MYOLO_REQUIRE(workspace_bytes >= myolo_det_loss_workspace_bytes(B, na, nl, ny, nx), "det_loss: workspace too small");
  cudaStream_t s = (cudaStream_t)stream;
  DetLossParams P;
  memset(&P, 0, sizeof(P));
  P.nl = nl; P.B = B; P.na = na; P.no = no; P.nc = no - 5; P.nt = nt; P.targets = targets;
  P.hyp_box = hyp_box; P.hyp_obj = hyp_obj; P.hyp_cls = hyp_cls; P.anchor_t = anchor_t; P.gr = gr; P.cp = cp; P.cn = cn;
  P.mult = mult; P.scale = scale_dev; P.items = items_out;
  unsigned char* w = reinterpret_cast<unsigned char*>(workspace);
  int64_t cells_total = 0;
  int max_cells = 0;
  for (int l = 0; l < nl; ++l) {
    P.p[l] = p[l]; P.dp[l] = dp[l]; P.ny[l] = ny[l]; P.nx[l] = nx[l]; P.balance[l] = balance[l];
    for (int k = 0; k < na * 2; ++k) P.anchors[l][k] = anchors_grid[l * na * 2 + k];
    const int cells = B * na * ny[l] * nx[l];
    max_cells = cells > max_cells ? cells : max_cells;
    cells_total += cells;
  }
  int64_t off = 0;
  for (int l = 0; l < nl; ++l) { P.winner[l] = reinterpret_cast<int*>(w + off); off += (int64_t)B * na * ny[l] * nx[l] * 4; }
  const int64_t tobj_off = off;
  for (int l = 0; l < nl; ++l) { P.tobj[l] = reinterpret_cast<float*>(w + off); off += (int64_t)B * na * ny[l] * nx[l] * 4; }
  P.nvalid = reinterpret_cast<int*>(w + off);
  P.sums = reinterpret_cast<float*>(w + off + 16);
  MYOLO_CHECK_CUDA(cudaMemsetAsync(w, 0xFF, (size_t)tobj_off, s));                       // winner = -1
  MYOLO_CHECK_CUDA(cudaMemsetAsync(w + tobj_off, 0, (size_t)(off - tobj_off) + 64, s));   // tobj = 0, counters = 0
  for (int l = 0; l < nl; ++l)
    MYOLO_CHECK_CUDA(cudaMemsetAsync(dp[l], 0, (size_t)B * na * ny[l] * nx[l] * no * sizeof(float), s));
  const int ncand = 5 * na * nt;
  if (ncand > 0) {
    const dim3 gc((unsigned)((ncand + 127) / 128), (unsigned)nl);
    det_assign_kernel<<<gc, 128, 0, s>>>(P);
    MYOLO_LAUNCH_CHECK();
    det_match_kernel<<<gc, 128, 0, s>>>(P);
    MYOLO_LAUNCH_CHECK();
  }
  const dim3 go((unsigned)std::min(296, (max_cells + 255) / 256), (unsigned)nl);
  det_obj_kernel<<<go, 256, 0, s>>>(P);
  MYOLO_LAUNCH_CHECK();
  det_items_kernel<<<1, 1, 0, s>>>(P);
  MYOLO_LAUNCH_CHECK();
  return 0;
}
