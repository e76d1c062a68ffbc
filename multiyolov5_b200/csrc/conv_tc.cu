// Fused Conv(+folded BN)+bias+SiLU(+residual) as an implicit GEMM on the Hopper tensor cores (wgmma), sm_90a.
//
//   D[128 pixels x BN channels] (fp32, registers)  +=  A[128 x kc] (NHWC activations, fp16)  *  B[BN x kc]^T (packed weights, fp16)
//
// * M tile  = a tw x th rectangle of output pixels of ONE image (tw*th = 128).  For every filter tap the A operand is the
//   same rectangle shifted by (dx,dy): one 4-D TMA box load {kc channels, tw, th, 1} with hardware zero fill at the
//   image border (that is the conv padding).  Stride-2 convs use four "parity" tensor maps (even/odd rows x cols)
//   so that the stride-2 gather is again a dense box.  No im2col buffer ever exists in HBM.
// * K loop  = taps x (Ci/kc) chunks, 64 K-elements per pipeline stage; operands are K-major with the 32/64/128-byte
//   TMA swizzle named in the wgmma shared-memory descriptor.
// * warp roles (384 threads = 3 warpgroups): warp 0 = TMA producer (one elected lane issues), warps 1-3 idle, warpgroups 1 and 2 =
//   consumers.  Consumer warpgroup w issues m64nBNk16 wgmma for pixel rows [64w, 64w+64) of the tile into its register accumulators,
//   releases each operand stage as soon as the MMAs that read it have retired, and runs the epilogue (bias, activation, residual,
//   fp16 / fp32 stores) straight from the accumulator fragment while the producer already fetches the next tile.
// * persistent grid (one CTA per SM, deep operand ring), programmatic dependent launch (prologue overlaps the previous kernel's tail).
//
// Reference semantics: Conv.fuseforward (reference models/common.py:45-46) with BN folded as in
// utils/torch_utils.py:182-202; Bottleneck shortcut add (models/common.py:105).
#include "conv.h"
#include "wgmma.cuh"

#ifndef MYOLO_SILU_SFU_EVERY
#define MYOLO_SILU_SFU_EVERY 2   // every n-th output channel of a 16-channel group takes the two-MUFU SiLU (balances the FMA pipe and the SFU)
#endif

namespace myolo {

static constexpr int kTileM = 128;
static constexpr int kKStage = 64;        // K elements per pipeline stage
static constexpr int kNumThreads = 384;   // producer warpgroup + two consumer warpgroups
static constexpr int kMaxStages = 8;
static constexpr int kSmemBudget = 227 * 1024;
static constexpr int kBiasBytes = 8192;   // bias vector of the layer in shared memory (<= 1920 output channels: the data gradient
                                          // of SPP.cv2 has 1024)

// K-major swizzled operand (rows of kc*2 bytes = the swizzle width, 8-row swizzle atoms), PTX ISA "matrix descriptor" of wgmma
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr, int row_bytes) {
  const uint64_t layout = row_bytes == 128 ? 1ull : (row_bytes == 64 ? 2ull : 3ull);
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);             // start address
  d |= (uint64_t)1 << 16;                              // leading byte offset (unused for swizzled K-major)
  d |= (uint64_t)((8u * row_bytes) >> 4) << 32;        // stride byte offset: next group of 8 rows
  d |= layout << 62;                                   // swizzle mode
  return d;
}

struct TileCoord { int b, y0, x0, n0; };
__device__ __forceinline__ int fdiv(int n, const FastDiv& f) { return (int)((__umulhi((unsigned)n, f.mul) + (unsigned)n) >> f.shr); }
__device__ __forceinline__ TileCoord decode_tile(const ConvTcParams& p, int tile, int tiles_per_img) {
  TileCoord t;
  const int m_tile = fdiv(tile, p.fd_ntn);
  const int n_tile = tile - m_tile * p.n_tiles_n;
  t.b = fdiv(m_tile, p.fd_tpi);
  const int r = m_tile - t.b * tiles_per_img;
  const int ty = fdiv(r, p.fd_tx);
  t.y0 = ty * p.th;
  t.x0 = (r - ty * p.tiles_x) * p.tw;
  t.n0 = n_tile * p.BN;
  return t;
}

__device__ __forceinline__ float act_out(float v, int act, int ch) {
  if (act == MYOLO_ACT_SILU) return (ch & 15) % MYOLO_SILU_SFU_EVERY == MYOLO_SILU_SFU_EVERY - 1 ? silu_f_sfu(v) : silu_f(v);
  if (act == MYOLO_ACT_SIGMOID) return sigmoid_f(v);
  return v;
}

// epilogue of one consumer warpgroup: the m64nBN accumulator fragment holds, for j < BN/8 and h < 2, output channels 8j + 2(lane%4) + {0,1}
// of tile row 16*(warp%4) + lane/4 + 8h, in acc[4j + 2h + {0,1}]
template <int BN, bool RES>
__device__ __forceinline__ void epilogue(const ConvTcParams& p, const float (&acc)[BN / 2], const float* bias_s, const TileCoord& tc, int row0) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    const int py = tc.y0 + (row >> p.log2_tw), px = tc.x0 + (row & (p.tw - 1));
    if (py >= p.Ho || px >= p.Wo) continue;
    const size_t pix = ((size_t)tc.b * p.Ho + py) * p.Wo + px;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      const int c = 8 * j + 2 * (lane & 3);
      const int n = tc.n0 + c;
      float v0 = act_out(acc[4 * j + 2 * h] + bias_s[n], p.act, c);
      float v1 = act_out(acc[4 * j + 2 * h + 1] + bias_s[n + 1], p.act, c + 1);
      if (p.out_mode == 0) {
        if (n >= p.out_c) continue;
        if (RES && n < p.Co) {
          const float2 r = __half22float2(*reinterpret_cast<const __half2*>(p.residual + pix * p.res_ctot + n));
          v0 += r.x;
          v1 += r.y;
        }
        *reinterpret_cast<__half2*>(p.out_f16 + pix * p.out_ctot + n) = __floats2half2_rn(v0, v1);
      } else if (n < p.out_ctot) {
        *reinterpret_cast<float2*>(p.out_f32 + pix * p.out_ctot + n) = make_float2(v0, v1);
      }
    }
  }
}

template <int BN, bool RES>
__global__ void __launch_bounds__(kNumThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmA3,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ConvTcParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int S = p.num_stages;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + S * p.a_stage_bytes;
  float* bias_s = reinterpret_cast<float*>(smem_b + S * p.b_stage_bytes);   // [n_tiles_n * BN] fp32
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(bias_s) + kBiasBytes);
  uint64_t* empty_bar = full_bar + S;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);   // warp-uniform for the compiler: wgmma is issued under role branches
  const int a_sub_bytes = kTileM * p.kc * 2;
  const int b_sub_bytes = BN * p.kc * 2;
  const int tiles_per_img = p.tiles_x * p.tiles_y;

  // programmatic dependent launch: let the next kernel of the stream start its own prologue as early as possible
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA0);
    tma_prefetch_desc(&tmB);
    for (int i = 0; i < S; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 2);          // one arrive per consumer warpgroup
    }
    fence_mbar_init();
  }
  if (threadIdx.x >= 128) {                 // the bias vector is a weight constant: copied before the dependency wait
    const int nb_tot = p.n_tiles_n * BN;
    for (int i = threadIdx.x - 128; i < nb_tot; i += kNumThreads - 128) bias_s[i] = __ldg(p.bias + i);
  }
  __syncthreads();

  if (warp == 0) {
    // ===================== TMA producer (warp-converged; one elected lane issues) =====================
    const bool leader = elect_one();
    asm volatile("griddepcontrol.wait;" ::: "memory");   // activations come from predecessor kernels
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile, tiles_per_img);
      int tap = 0, cb = 0, q = 0;
      for (int ks = 0; ks < p.n_kstages; ++ks) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        __syncwarp();
        const int nch = min(p.chunks_per_stage, p.n_chunks - q);
        if (leader) mbar_arrive_expect_tx(&full_bar[stage], nch * (a_sub_bytes + b_sub_bytes));
        uint8_t* sa = smem_a + stage * p.a_stage_bytes;
        uint8_t* sb = smem_b + stage * p.b_stage_bytes;
        for (int j = 0; j < nch; ++j, ++q) {
          const int mi = p.tap_map[tap];
          const CUtensorMap* tm = mi == 0 ? &tmA0 : (mi == 1 ? &tmA1 : (mi == 2 ? &tmA2 : &tmA3));
          if (leader) {
            tma_load_4d(sa + j * a_sub_bytes, tm, &full_bar[stage], cb * p.kc, t.x0 + p.tap_dx[tap], t.y0 + p.tap_dy[tap], t.b);
            tma_load_2d(sb + j * b_sub_bytes, &tmB, &full_bar[stage], q * p.kc, t.n0);
          }
          if (++cb == p.cblocks) { cb = 0; ++tap; }
        }
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
    }
  } else if (warp >= 4) {
    // ===================== consumers: two warpgroups, 64 pixel rows each =====================
    const int cw = (warp >> 2) - 1;
    const bool signaller = (threadIdx.x & 127) == 0;
    const int row_bytes = p.kc * 2;
    const int kmma = p.kc / 16;
    if (RES) asm volatile("griddepcontrol.wait;" ::: "memory");   // the residual is a predecessor's output
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t a_base = smem_u32(smem_a) + (uint32_t)(cw * 64 * row_bytes);
    const uint32_t b_base = smem_u32(smem_b);
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile, tiles_per_img);
      int q = 0, prev = -1;
      for (int ks = 0; ks < p.n_kstages; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const int nch = min(p.chunks_per_stage, p.n_chunks - q);
        const uint32_t sa = a_base + (uint32_t)(stage * p.a_stage_bytes);
        const uint32_t sb = b_base + (uint32_t)(stage * p.b_stage_bytes);
        wgmma_fence();
        wgmma_fence_regs(acc);
        for (int j = 0; j < nch; ++j)
          for (int k = 0; k < kmma; ++k)      // 16 K-elements = 32 bytes further inside the swizzle atom
            wgmma_f16<BN, 0, 0>(acc, make_smem_desc(sa + j * a_sub_bytes + 32 * k, row_bytes),
                                make_smem_desc(sb + j * b_sub_bytes + 32 * k, row_bytes), (uint32_t)((ks | j | k) != 0));
        wgmma_commit();
        wgmma_wait<1>();                        // the previous stage's MMAs have retired: its operands may be overwritten
        if (prev >= 0 && signaller) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        q += nch;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && signaller) mbar_arrive(&empty_bar[prev]);
      epilogue<BN, RES>(p, acc, bias_s, t, cw * 64 + (warp & 3) * 16);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

static int encode_map(CUtensorMap* m, int rank, void* addr, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, int swizzle_bytes) {
  PFN_encodeTiled enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return MYOLO_E_CUDA;
  }
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                          : swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                          : swizzle_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B
                                                : CU_TENSOR_MAP_SWIZZLE_NONE;
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, addr, gd, gs, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u sw %d", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)(rank > 2 ? dims[2] : 0),
              (unsigned long long)(rank > 3 ? dims[3] : 0), box[0], box[1], rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0,
              swizzle_bytes);
    return MYOLO_E_CUDA;
  }
  return 0;
}

int encode_tensor_map(CUtensorMap* m, int rank, void* addr, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                      int swizzle_bytes) {
  return encode_map(m, rank, addr, dims, strides_bytes, box, swizzle_bytes);
}

static void choose_tile(int W, int H, int* tw, int* th) {
  long best = -1;
  for (int t = 128; t >= 8; t >>= 1) {
    const int hh = 128 / t;
    const long tiles = (long)ceil_div(W, t) * ceil_div(H, hh);
    if (best < 0 || tiles < best) {
      best = tiles;
      *tw = t;
      *th = hh;
    }
  }
}

bool conv_tc_eligible(const ConvOp& op) {
  if (op.in.dtype != MYOLO_F16) return false;
  if (op.Ci_pad % 16 != 0 || op.in.C != op.Ci_pad) return false;
  if (!(op.k == 1 || op.k == 3)) return false;
  if (!(op.stride == 1 || (op.stride == 2 && op.k == 3 && op.dil == 1))) return false;
  if (op.stride == 2 && ((op.in.H | op.in.W) & 1)) return false;
  if (op.in.ctot % 8 != 0) return false;
  if (op.out.dtype == MYOLO_F16) {
    if (op.out.C % 8 != 0 || op.out.ctot % 8 != 0) return false;
    if (op.has_res && (op.res.dtype != MYOLO_F16 || op.res.ctot % 8 != 0 || op.Co % 16 != 0)) return false;
  } else {
    if (op.has_res || op.out.ctot % 4 != 0) return false;
  }
  // tiny maps run on the generic kernel (TMA boxes larger than the tensor are avoided on purpose)
  if (op.out.W < 8 || op.out.H < 2 || op.out.W * op.out.H < 128) return false;
  if (align_up(op.Co, 16) * 4 + 512 > kBiasBytes) return false;   // the bias vector lives in shared memory
  return true;
}

int conv_tc_prepare(ConvOp& op, int num_sms) {
  ConvTcParams& p = op.p;
  memset(&p, 0, sizeof(p));
  auto ilog2 = [](int v) { int l = 0; while ((1 << l) < v) ++l; return l; };
  const int Ho = op.out.H, Wo = op.out.W;
  p.B = op.in.B;
  p.Ho = Ho;
  p.Wo = Wo;
  choose_tile(Wo, Ho, &p.tw, &p.th);
  p.log2_tw = ilog2(p.tw);
  p.tiles_x = ceil_div(Wo, p.tw);
  p.tiles_y = ceil_div(Ho, p.th);
  p.Co = op.Co;
  // N tile: whole Co if it fits in 128, else the largest multiple of 16 <= 128 dividing Co16 (Co_pad sized by the caller)
  const int co16 = (int)align_up(op.Co, 16);
  p.BN = co16 <= 128 ? co16 : 128;
  if (co16 > 128 && co16 % 128 != 0) {
    for (int bn = 128; bn >= 16; bn -= 16)
      if (co16 % bn == 0) { p.BN = bn; break; }
  }
  p.n_tiles_n = ceil_div(co16, p.BN);
  MYOLO_REQUIRE(op.Co_pad >= p.n_tiles_n * p.BN, "conv_tc: Co_pad %d < %d", op.Co_pad, p.n_tiles_n * p.BN);
  p.total_tiles = p.B * p.tiles_x * p.tiles_y * p.n_tiles_n;
  p.kc = op.Ci_pad % 64 == 0 ? 64 : (op.Ci_pad % 32 == 0 ? 32 : 16);
  p.cblocks = op.Ci_pad / p.kc;
  p.taps = op.k * op.k;
  p.n_chunks = p.taps * p.cblocks;
  p.chunks_per_stage = kKStage / p.kc;
  p.n_kstages = ceil_div(p.n_chunks, p.chunks_per_stage);
  p.act = op.act;
  p.bias = op.bias;
  p.residual = op.has_res ? reinterpret_cast<const __half*>(op.res.base) : nullptr;
  p.res_ctot = op.has_res ? op.res.ctot : 0;
  p.out_mode = op.out.dtype == MYOLO_F16 ? 0 : 1;
  p.out_f16 = p.out_mode ? nullptr : reinterpret_cast<__half*>(op.out.base);
  p.out_f32 = p.out_mode ? reinterpret_cast<float*>(op.out.base) : nullptr;
  p.out_c = op.out.C;
  p.out_ctot = op.out.ctot;
  for (int t = 0; t < p.taps; ++t) {
    const int ky = op.k == 3 ? t / 3 : 1, kx = op.k == 3 ? t % 3 : 1;
    if (op.stride == 1) {
      p.tap_map[t] = 0;
      p.tap_dx[t] = (kx - 1) * op.dil;
      p.tap_dy[t] = (ky - 1) * op.dil;
    } else {  // stride 2, k 3, pad 1: input row = 2*oy + ky - 1
      const int pyb = (ky == 1) ? 0 : 1, pxb = (kx == 1) ? 0 : 1;
      p.tap_map[t] = pyb * 2 + pxb;
      p.tap_dy[t] = (ky == 0) ? -1 : 0;
      p.tap_dx[t] = (kx == 0) ? -1 : 0;
    }
  }
  p.fd_ntn = make_fastdiv((unsigned)p.n_tiles_n);
  p.fd_tpi = make_fastdiv((unsigned)(p.tiles_x * p.tiles_y));
  p.fd_tx = make_fastdiv((unsigned)p.tiles_x);
  // stage geometry: one CTA per SM with as deep an operand ring as shared memory allows
  p.a_stage_bytes = kTileM * kKStage * 2;
  p.b_stage_bytes = (int)align_up(p.BN * kKStage * 2, 1024);
  const int stage_bytes = p.a_stage_bytes + p.b_stage_bytes;
  const int misc = 1024 /*barriers*/ + kBiasBytes + 1024 /*alignment slack*/;
  int S = (kSmemBudget - misc) / stage_bytes;
  if (S > kMaxStages) S = kMaxStages;
  MYOLO_REQUIRE(S >= 2, "conv_tc: not enough shared memory for 2 stages");
  MYOLO_REQUIRE(p.n_tiles_n * p.BN * 4 <= kBiasBytes, "conv_tc: %d output channels exceed the shared-memory bias buffer", p.n_tiles_n * p.BN);
  p.num_stages = S;
  op.smem = S * stage_bytes + misc;
  op.grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;

  // ---- tensor maps ----
  const int esz = 2;
  const int sw = p.kc * 2;
  const TensorView& in = op.in;
  if (op.stride == 1) {
    uint64_t dims[4] = {(uint64_t)in.C, (uint64_t)in.W, (uint64_t)in.H, (uint64_t)in.B};
    uint64_t str[3] = {(uint64_t)in.ctot * esz, (uint64_t)in.W * in.ctot * esz, (uint64_t)in.H * in.W * in.ctot * esz};
    uint32_t box[4] = {(uint32_t)p.kc, (uint32_t)p.tw, (uint32_t)p.th, 1};
    int rc = encode_map(&op.tmA[0], 4, in.base, dims, str, box, sw);
    if (rc) return rc;
    op.tmA[1] = op.tmA[2] = op.tmA[3] = op.tmA[0];
  } else {
    for (int py = 0; py < 2; ++py)
      for (int px = 0; px < 2; ++px) {
        uint64_t dims[4] = {(uint64_t)in.C, (uint64_t)in.W / 2, (uint64_t)in.H / 2, (uint64_t)in.B};
        uint64_t str[3] = {(uint64_t)2 * in.ctot * esz, (uint64_t)2 * in.W * in.ctot * esz,
                           (uint64_t)in.H * in.W * in.ctot * esz};
        uint32_t box[4] = {(uint32_t)p.kc, (uint32_t)p.tw, (uint32_t)p.th, 1};
        void* base = reinterpret_cast<__half*>(in.base) + ((size_t)py * in.W + px) * in.ctot;
        int rc = encode_map(&op.tmA[py * 2 + px], 4, base, dims, str, box, sw);
        if (rc) return rc;
      }
  }
  {
    const uint64_t Kt = (uint64_t)p.taps * op.Ci_pad;
    uint64_t dims[2] = {Kt, (uint64_t)op.Co_pad};
    uint64_t str[1] = {Kt * esz};
    uint32_t box[2] = {(uint32_t)p.kc, (uint32_t)p.BN};
    int rc = encode_map(&op.tmB, 2, const_cast<__half*>(op.w), dims, str, box, sw);
    if (rc) return rc;
  }
  return 0;
}

template <int BN, bool RES>
static cudaError_t launch_bn(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<BN, RES>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel<BN, RES>, op.tmA[0], op.tmA[1], op.tmA[2], op.tmA[3], op.tmB, op.p);
}

template <bool RES>
static cudaError_t launch_res(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  switch (op.p.BN) {
    case 16: return launch_bn<16, RES>(op, cfg);
    case 32: return launch_bn<32, RES>(op, cfg);
    case 48: return launch_bn<48, RES>(op, cfg);
    case 64: return launch_bn<64, RES>(op, cfg);
    case 80: return launch_bn<80, RES>(op, cfg);
    case 96: return launch_bn<96, RES>(op, cfg);
    case 112: return launch_bn<112, RES>(op, cfg);
    case 128: return launch_bn<128, RES>(op, cfg);
  }
  return cudaErrorInvalidValue;
}

int conv_tc_launch(const ConvOp& op, cudaStream_t stream) {
  MYOLO_REQUIRE(op.p.BN % 16 == 0 && op.p.BN >= 16 && op.p.BN <= 128, "conv_tc: unsupported N tile %d", op.p.BN);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(op.grid);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = op.smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  MYOLO_CHECK_CUDA(op.p.residual != nullptr ? launch_res<true>(op, cfg) : launch_res<false>(op, cfg));
  g_launch_count++;
  return 0;
}

}  // namespace myolo
