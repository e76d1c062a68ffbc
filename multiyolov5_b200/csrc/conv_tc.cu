// Fused Conv(+folded BN)+bias+SiLU(+residual) as an implicit GEMM on the Hopper tensor cores (wgmma), sm_90a.
//
//   D[128 pixels x BN channels] (fp32, registers)  +=  A[128 x kc] (NHWC activations, fp16)  *  B[BN x kc]^T (packed weights, fp16)
//
// * M tile  = a tw x th rectangle of output pixels of ONE image (tw*th = 128).  For every filter tap the A operand is the
//   same rectangle shifted by (dx,dy): one 4-D TMA box load {kc channels, tw, th, 1} with hardware zero fill at the
//   image border (that is the conv padding).  Stride-2 convs use four "parity" tensor maps (even/odd rows x cols)
//   so that the stride-2 gather is again a dense box.  No im2col buffer ever exists in HBM.
// * K loop  = taps x (Ci/kc) chunks, 64 K-elements per pipeline stage; operands are K-major with the 32/64/128-byte
//   TMA swizzle named in the wgmma shared-memory descriptor.  kc is a template parameter, so the MMAs of a stage are one
//   straight-line block and one wgmma group.
// * operand reuse: a weight slice that fits next to six A stages stays resident for the CTA's whole persistent loop, and 3x3 stride-1
//   layers with resident weights load one strip {kc, tw + 2 dil, th, 1} per filter row that serves its three kx taps (conv_tc_prepare).
// * warp roles (384 threads = 3 warpgroups): warp 0 = TMA producer (one elected lane issues), warps 1-3 idle, warpgroups 1 and 2 =
//   consumers.  Consumer warpgroup w issues m64nBNk16 wgmma for pixel rows [64w, 64w+64) of the tile into its register accumulators,
//   releases each operand stage as soon as the MMAs that read it have retired, and runs the epilogue (bias, activation, residual,
//   fp16 / fp32 stores) from the accumulator registers while the producer already fetches the next tile; fp16 tiles are written as
//   16-byte vectors of 8 channels after a transpose within each quad of lanes (epilogue()).
// * persistent grid (one CTA per SM with a deep operand ring, or two with resident weights and BN <= 64 where half the shared memory
//   still holds a useful ring, see conv_tc_prepare), programmatic dependent launch (prologue overlaps the previous kernel's tail).
//   At two CTAs per SM the producer warpgroup hands its registers to the consumers (setmaxnreg).
//
// Reference semantics: Conv.fuseforward (reference models/common.py:45-46) with BN folded as in
// utils/torch_utils.py:182-202; Bottleneck shortcut add (models/common.py:105).
#include "conv.h"
#include "wgmma.cuh"

namespace myolo {

static constexpr int kTileM = 128;
static constexpr int kKStage = 64;        // K elements per pipeline stage
static constexpr int kNumThreads = 384;   // producer warpgroup + two consumer warpgroups
static constexpr int kMaxStages = 8;
static constexpr int kMinResidentStages = 6;   // A stages a layer keeps next to resident weights (with 4, the 144 KB pack of the
                                               // 3x3 s2 64->128 layer left 4 stages and ran 5 us slower than streamed with 6)
static constexpr int kMaxStripBlocks = 4;      // channel blocks of a strip-mode layer (mma_strip_row instantiations)
static constexpr int kSmemBudget = 227 * 1024;
static constexpr int kSmemBudgetTwoCtas = 228 * 1024 / 2 - 1024;   // per CTA when two share an SM (228 KB, 1 KB reserved per CTA)
static constexpr int kMinTwoCtaStages = 4;       // A stages per CTA at two CTAs per SM on the per-tap path (strip mode: 2 strip stages)
static constexpr int kTwoCtaMaxBN = 64;          // widest N tile whose consumers fit kConsumerRegs (BN / 2 accumulators + residual vectors)
static constexpr int kProducerRegs = 24;         // setmaxnreg at two CTAs per SM: 128 x 24 + 256 x 104 <= 384 x 80, the pool of one CTA
static constexpr int kConsumerRegs = 104;
static constexpr int kMaxBiasBytes = 12288;      // bias vector of the layer in shared memory (<= 2944 output channels: the data gradient
                                                 // of SPP.cv2 has 4 c_ = 1024 / 1536 / 2048 / 2560 in s / m / l / x).  The shared-memory
                                                 // layout is sized per layer (size_launch), so a layer of at most 1920 channels is
                                                 // launched exactly as it was under the former 8 KB bound
// weight packs up to this size stay resident: 121 KB, room for kMinResidentStages A stages and 10 KB of barriers, a bias vector of up to
// 1920 channels and slack (a wider layer keeps one A stage fewer; the 128 KB packs measured the same resident or streamed, DESIGN §5)
static constexpr int kResidentPackLimit = kSmemBudget - 10 * 1024 - kMinResidentStages * kTileM * kKStage * 2;
static constexpr int kSiluSfuEvery = 2;   // every n-th output channel of a 16-channel group takes the two-MUFU SiLU (balances the FMA
                                          // pipe and the SFU)

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

// register reallocation between warpgroups (every warp of the warpgroup executes the same instruction)
template <int N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <int N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }

__device__ __forceinline__ float act_out(float v, int act, int ch) {
  if (act == MYOLO_ACT_SILU) return (ch & 15) % kSiluSfuEvery == kSiluSfuEvery - 1 ? silu_f_sfu(v) : silu_f(v);
  if (act == MYOLO_ACT_SIGMOID) return sigmoid_f(v);
  return v;
}

// The m64nBN accumulator fragment holds, for j < BN/8 and h < 2, output channels 8j + 2(lane%4) + {0,1} of tile row
// 16*(warp%4) + lane/4 + 8h, in acc[4j + 2h + {0,1}]: the four lanes of a quad share a row, and lane q holds 32-bit word q (two fp16
// channels) of every 8-channel group j.  The fp16 epilogue transposes each 4x4 block of words (groups 4g .. 4g+3) within the quad, so
// that lane q owns all 8 channels of group 4g + q and writes them with one 16-byte store: a warp instruction then covers 64 contiguous
// bytes in each of 8 rows instead of 16.  A last block of two groups (BN % 32 == 16) is padded with zero words that no lane stores.
template <int BN>
struct EpiGroups { static constexpr int n = (BN + 31) / 32; };

// before: lane q of the quad holds w[i] = word q of group i; after: w[i] = word i of group q.  Two butterfly steps (lane masks 1 and 2);
// in each, a lane keeps the words whose index agrees with its own lane bit and trades the other two with its partner.  Every lane of
// the warp takes part (full mask): callers run it before any per-row early exit.
__device__ __forceinline__ void quad_transpose(uint32_t (&w)[4]) {
  const int q = threadIdx.x & 3;
#pragma unroll
  for (int m = 1; m <= 2; m <<= 1) {
    const bool hi = (q & m) != 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (i & m) continue;
      const uint32_t recv = __shfl_xor_sync(0xffffffffu, hi ? w[i] : w[i | m], m);
      if (hi) w[i] = recv;
      else w[i | m] = recv;
    }
  }
}

// the residual values of the thread's epilogue, all loads in flight at once, each one 16-byte vector: the 8 channels of group 4g + lane%4
// that this lane will store (so an output aliasing the residual, as in the data-gradient convs, is read and written by the same lane,
// and all of the warp's loads are issued before its first store).  Issued before the tile's last MMAs retire.
template <int BN>
__device__ __forceinline__ void load_residual(const ConvTcParams& p, const TileCoord& tc, int row0, uint4 (&res)[2][EpiGroups<BN>::n]) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    const int py = tc.y0 + (row >> p.log2_tw), px = tc.x0 + (row & (p.tw - 1));
    const bool in_map = py < p.Ho && px < p.Wo;
    const size_t pix = ((size_t)tc.b * p.Ho + py) * p.Wo + px;
#pragma unroll
    for (int g = 0; g < EpiGroups<BN>::n; ++g) {
      const int j = 4 * g + (lane & 3);
      const int n = tc.n0 + 8 * j;
      res[h][g] = in_map && j < BN / 8 && n < p.out_c && n < p.Co ? *reinterpret_cast<const uint4*>(p.residual + pix * p.res_ctot + n)
                                                                  : make_uint4(0u, 0u, 0u, 0u);
    }
  }
}

__device__ __forceinline__ uint32_t half2_bits(__half2 v) { return *reinterpret_cast<uint32_t*>(&v); }
__device__ __forceinline__ __half2 bits_half2(uint32_t v) { return *reinterpret_cast<__half2*>(&v); }

// epilogue of one consumer warpgroup: bias, activation, residual (fp32, before the single fp16 rounding), stores into the output slice
template <int BN, bool RES>
__device__ __forceinline__ void epilogue(const ConvTcParams& p, const float (&acc)[BN / 2], uint4 (&res)[2][EpiGroups<BN>::n],
                                         const float* bias_s, const TileCoord& tc, int row0) {
  const int lane = threadIdx.x & 31;
  const int q = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int row = row0 + (lane >> 2) + 8 * h;
    const int py = tc.y0 + (row >> p.log2_tw), px = tc.x0 + (row & (p.tw - 1));
    const bool in_map = py < p.Ho && px < p.Wo;   // uniform over the quad: the transposes below run for every row regardless
    const size_t pix = ((size_t)tc.b * p.Ho + py) * p.Wo + px;
    if (p.out_mode == 0) {
#pragma unroll
      for (int g = 0; g < EpiGroups<BN>::n; ++g) {
        uint32_t r[4] = {0u, 0u, 0u, 0u};
        if constexpr (RES) {                   // back to the fragment layout: r[i] = this lane's two channels of group 4g + i
          r[0] = res[h][g].x;
          r[1] = res[h][g].y;
          r[2] = res[h][g].z;
          r[3] = res[h][g].w;
          quad_transpose(r);
        }
        uint32_t w[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int j = 4 * g + i;
          w[i] = 0u;
          if (j < BN / 8) {
            const int c = 8 * j + 2 * q;
            const int n = tc.n0 + c;
            float v0 = act_out(acc[4 * j + 2 * h] + bias_s[n], p.act, c);
            float v1 = act_out(acc[4 * j + 2 * h + 1] + bias_s[n + 1], p.act, c + 1);
            if (RES && n < p.Co) {
              const float2 rf = __half22float2(bits_half2(r[i]));
              v0 += rf.x;
              v1 += rf.y;
            }
            w[i] = half2_bits(__floats2half2_rn(v0, v1));
          }
        }
        quad_transpose(w);                     // w = the 8 channels of group 4g + q
        const int j = 4 * g + q;
        const int n = tc.n0 + 8 * j;
        if (in_map && j < BN / 8 && n < p.out_c)
          *reinterpret_cast<uint4*>(p.out_f16 + pix * p.out_ctot + n) = make_uint4(w[0], w[1], w[2], w[3]);
      }
    } else if (in_map) {
      const int n_end = min(p.out_c, p.Co);   // the conv's channels inside the slice: never its neighbours or a buffer's padding
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + 2 * q;
        const int n = tc.n0 + c;
        const float v0 = act_out(acc[4 * j + 2 * h] + bias_s[n], p.act, c);
        const float v1 = act_out(acc[4 * j + 2 * h + 1] + bias_s[n + 1], p.act, c + 1);
        float* dst = p.out_f32 + pix * p.out_ctot + n;
        if (n + 1 < n_end) *reinterpret_cast<float2*>(dst) = make_float2(v0, v1);
        else if (n < n_end) *dst = v0;
      }
    }
  }
}

// the MMAs of one operand stage that holds NCH K chunks of KC channels, committed as ONE wgmma group.  Fence, MMAs and commit sit in
// one straight-line block: with a runtime trip count, or a commit behind a branch, ptxas closes a group after every loop body and
// turns the commit into an empty group, so waiting for "all but the newest group" drains the tensor pipe once per stage.
template <int KC, int BN, int NCH>
__device__ __forceinline__ void mma_stage(float (&acc)[BN / 2], uint32_t sa, uint32_t sb, uint32_t scale_first) {
  constexpr int kRowBytes = KC * 2;
  wgmma_fence();
  wgmma_fence_regs(acc);
#pragma unroll
  for (int j = 0; j < NCH; ++j)
#pragma unroll
    for (int k = 0; k < KC / 16; ++k)      // 16 K-elements = 32 bytes further inside the swizzle atom
      wgmma_f16<BN, 0, 0>(acc, make_smem_desc(sa + j * (kTileM * KC * 2) + 32 * k, kRowBytes),
                          make_smem_desc(sb + j * (BN * KC * 2) + 32 * k, kRowBytes), (j | k) != 0 ? 1u : scale_first);
  wgmma_commit();
}

// strip mode: the MMAs of one filter row ky, its three kx taps x CB channel blocks in the K order of the per-tap path (taps outer,
// channel blocks inner), one wgmma group.  Tap kx reads the strip dx_bytes * kx further on: a start address off the 8-row swizzle
// atom is fine, since wgmma applies the swizzle to absolute shared-memory address bits as TMA does (matrix base offset stays 0).
template <int KC, int BN, int CB>
__device__ __forceinline__ void mma_strip_row(float (&acc)[BN / 2], uint32_t sa, uint32_t sb, uint32_t strip_sub_bytes, uint32_t dx_bytes,
                                              uint32_t scale_first) {
  constexpr int kRowBytes = KC * 2;
  wgmma_fence();
  wgmma_fence_regs(acc);
#pragma unroll
  for (int kx = 0; kx < 3; ++kx)
#pragma unroll
    for (int c = 0; c < CB; ++c)
#pragma unroll
      for (int k = 0; k < KC / 16; ++k)
        wgmma_f16<BN, 0, 0>(acc, make_smem_desc(sa + kx * dx_bytes + c * strip_sub_bytes + 32 * k, kRowBytes),
                            make_smem_desc(sb + (kx * CB + c) * (BN * KC * 2) + 32 * k, kRowBytes), (kx | c | k) != 0 ? 1u : scale_first);
  wgmma_commit();
}

template <int KC, int BN, bool RES, int CTAS_PER_SM>
__global__ void __launch_bounds__(kNumThreads, CTAS_PER_SM)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
               const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmA3,
               const __grid_constant__ CUtensorMap tmB, const __grid_constant__ ConvTcParams p) {
  constexpr int kChunksPerStage = kKStage / KC;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  const int S = p.num_stages;
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem_a + S * p.a_stage_bytes;                         // resident: K chunk q in slot q; else one ring stage per A stage
  float* bias_s = reinterpret_cast<float*>(smem_b + p.b_bytes);           // [n_tiles_n * BN] fp32
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(bias_s) + p.bias_bytes);
  uint64_t* empty_bar = full_bar + S;

  const int warp = __shfl_sync(0xffffffffu, threadIdx.x >> 5, 0);   // warp-uniform for the compiler: wgmma is issued under role branches
  constexpr int a_sub_bytes = kTileM * KC * 2;
  constexpr int b_sub_bytes = BN * KC * 2;
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

  if (warp < 4) {
    // ===================== TMA producer (warp 0, warp-converged; one elected lane issues) =====================
    if constexpr (CTAS_PER_SM == 2) setmaxnreg_dec<kProducerRegs>();   // warps 1-3 take part, then leave
    if (warp != 0) return;
    const bool leader = elect_one();
    // Activations come from predecessor kernels.  The weights are loaded after this wait as well: the training step repacks them
    // (myolo_plan_repack_weights) on the same stream before the forward, and only this wait orders that repack before the loads.
    asm volatile("griddepcontrol.wait;" ::: "memory");
    int stage = 0;
    uint32_t phase = 0;
    const int n_units = p.strip ? 3 : p.n_kstages;
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile, tiles_per_img);
      // resident weights: the first tile fills the slots as its K loop reaches them (gridDim.x is a multiple of n_tiles_n, so every
      // tile of this CTA has the same N tile); later tiles load A only
      const bool load_b = !p.resident || tile == (int)blockIdx.x;
      int tap = 0, cb = 0, q = 0;
      for (int ks = 0; ks < n_units; ++ks) {
        mbar_wait(&empty_bar[stage], phase ^ 1);
        __syncwarp();
        if (p.strip) {   // stage = filter row ks: one strip per channel block (x0 - dil .. x0 + tw + dil), weights of its 3 taps
          const int nq = 3 * p.cblocks;
          if (leader) {
            mbar_arrive_expect_tx(&full_bar[stage], p.cblocks * p.strip_box_bytes + (load_b ? nq * b_sub_bytes : 0));
            uint8_t* sa = smem_a + stage * p.a_stage_bytes;
            for (int c = 0; c < p.cblocks; ++c)
              tma_load_4d(sa + c * p.strip_sub_bytes, &tmA0, &full_bar[stage], c * KC, t.x0 - p.dil, t.y0 + (ks - 1) * p.dil, t.b);
            if (load_b)
              for (int j = ks * nq; j < (ks + 1) * nq; ++j) tma_load_2d(smem_b + j * b_sub_bytes, &tmB, &full_bar[stage], j * KC, t.n0);
          }
          if (++stage == S) { stage = 0; phase ^= 1; }
          continue;
        }
        const int nch = min(kChunksPerStage, p.n_chunks - q);
        if (leader) mbar_arrive_expect_tx(&full_bar[stage], nch * (a_sub_bytes + (load_b ? b_sub_bytes : 0)));
        uint8_t* sa = smem_a + stage * p.a_stage_bytes;
        uint8_t* sb = p.resident ? smem_b + q * b_sub_bytes : smem_b + stage * p.b_stage_bytes;
        for (int j = 0; j < nch; ++j, ++q) {
          const int mi = p.tap_map[tap];
          const CUtensorMap* tm = mi == 0 ? &tmA0 : (mi == 1 ? &tmA1 : (mi == 2 ? &tmA2 : &tmA3));
          if (leader) {
            tma_load_4d(sa + j * a_sub_bytes, tm, &full_bar[stage], cb * KC, t.x0 + p.tap_dx[tap], t.y0 + p.tap_dy[tap], t.b);
            if (load_b) tma_load_2d(sb + j * b_sub_bytes, &tmB, &full_bar[stage], q * KC, t.n0);
          }
          if (++cb == p.cblocks) { cb = 0; ++tap; }
        }
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
    }
  } else {
    // ===================== consumers: two warpgroups, 64 pixel rows each =====================
    if constexpr (CTAS_PER_SM == 2) setmaxnreg_inc<kConsumerRegs>();
    const int cw = (warp >> 2) - 1;
    const bool signaller = (threadIdx.x & 127) == 0;
    if (RES) asm volatile("griddepcontrol.wait;" ::: "memory");   // the residual is a predecessor's output
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    int stage = 0;
    uint32_t phase = 0;
    const uint32_t a_base = smem_u32(smem_a) + (uint32_t)(cw * 64 * KC * 2);
    const uint32_t b_base = smem_u32(smem_b);
    const int n_full = p.n_chunks / kChunksPerStage;     // stages with kChunksPerStage chunks; a last one holds the remaining chunks
    const int n_tail = p.n_chunks - n_full * kChunksPerStage;
    const int n_units = p.strip ? 3 : p.n_kstages;
    // strip mode: this warpgroup's 64 output pixels start at strip row (64 cw) mod tw, in strip line (64 cw) / tw
    const uint32_t strip_base = smem_u32(smem_a) + (uint32_t)((((cw * 64) & (p.tw - 1)) + ((cw * 64) >> p.log2_tw) * p.strip_w) * KC * 2);
    for (int tile = blockIdx.x; tile < p.total_tiles; tile += gridDim.x) {
      const TileCoord t = decode_tile(p, tile, tiles_per_img);
      int prev = -1;
      for (int ks = 0; ks < n_units; ++ks) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t scale_first = ks != 0;
        if (p.strip) {
          const uint32_t sa = strip_base + (uint32_t)(stage * p.a_stage_bytes);
          const uint32_t sb = b_base + (uint32_t)(ks * 3 * p.cblocks * b_sub_bytes);
          const uint32_t dx = (uint32_t)(p.dil * KC * 2), ss = (uint32_t)p.strip_sub_bytes;
          switch (p.cblocks) {
            case 1: mma_strip_row<KC, BN, 1>(acc, sa, sb, ss, dx, scale_first); break;
            case 2: mma_strip_row<KC, BN, 2>(acc, sa, sb, ss, dx, scale_first); break;
            case 3: mma_strip_row<KC, BN, 3>(acc, sa, sb, ss, dx, scale_first); break;
            default: mma_strip_row<KC, BN, 4>(acc, sa, sb, ss, dx, scale_first); break;
          }
        } else {
          const uint32_t sa = a_base + (uint32_t)(stage * p.a_stage_bytes);
          const uint32_t sb = b_base + (uint32_t)(p.resident ? ks * (kChunksPerStage * b_sub_bytes) : stage * p.b_stage_bytes);
          if (kChunksPerStage == 1 || ks < n_full) {
            mma_stage<KC, BN, kChunksPerStage>(acc, sa, sb, scale_first);
          } else if constexpr (kChunksPerStage > 1) {
            if (n_tail == 1) mma_stage<KC, BN, 1>(acc, sa, sb, scale_first);
            if constexpr (kChunksPerStage > 2) {
              if (n_tail == 2) mma_stage<KC, BN, 2>(acc, sa, sb, scale_first);
              if (n_tail == 3) mma_stage<KC, BN, 3>(acc, sa, sb, scale_first);
            }
          }
        }
        wgmma_wait<1>();                        // the previous stage's MMAs have retired: its operands may be overwritten
        if (prev >= 0 && signaller) mbar_arrive(&empty_bar[prev]);
        prev = stage;
        if (++stage == S) { stage = 0; phase ^= 1; }
      }
      const int row0 = cw * 64 + (warp & 3) * 16;
      uint4 res[2][EpiGroups<BN>::n];
      if constexpr (RES) load_residual<BN>(p, t, row0, res);
      wgmma_wait<0>();
      wgmma_fence_regs(acc);
      if (prev >= 0 && signaller) mbar_arrive(&empty_bar[prev]);
      epilogue<BN, RES>(p, acc, res, bias_s, t, row0);
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
    // the epilogue stores (and loads the residual in) 16-byte vectors of 8 channels: the slices must start on a 16-byte boundary
    auto aligned16 = [](const void* ptr) { return reinterpret_cast<uintptr_t>(ptr) % 16 == 0; };
    if (op.out.C % 8 != 0 || op.out.ctot % 8 != 0 || !aligned16(op.out.base)) return false;
    if (op.has_res && (op.res.dtype != MYOLO_F16 || op.res.ctot % 8 != 0 || op.Co % 16 != 0 || !aligned16(op.res.base))) return false;
  } else {
    // the epilogue stores two channels as one 8-byte vector (an odd last channel alone): the slice must start on an 8-byte boundary
    if (op.has_res || op.out.ctot % 4 != 0 || reinterpret_cast<uintptr_t>(op.out.base) % 8 != 0) return false;
  }
  // tiny maps run on the generic kernel (TMA boxes larger than the tensor are avoided on purpose)
  if (op.out.W < 8 || op.out.H < 2 || op.out.W * op.out.H < 128) return false;
  if (align_up(op.Co, 16) * 4 + 512 > kMaxBiasBytes) return false;   // the bias vector lives in shared memory
  return true;
}

// N tile bn and what follows from it: tile count, residency, strip mode, CTAs per SM, stage count, grid and shared memory.  Returns the
// CTAs per SM.
//
// One CTA per SM gets as deep an operand ring as shared memory allows.  The weight slice of one N tile stays resident when it is at most
// kResidentPackLimit and every CTA of the persistent grid keeps one N tile (grid % n_tiles_n == 0): a CTA then reads its weights from L2
// once instead of once per tile.  Strip mode (3x3 stride 1 with resident weights, tw >= 64 so that each consumer's 64 pixels lie in one
// strip line): a stage holds one filter row's strips of all channel blocks; at least two such stages must fit.
//
// Two CTAs per SM: with resident weights, BN <= kTwoCtaMaxBN and more tiles than SMs, a second CTA on each SM overlaps its waits and MMAs
// with the first one's epilogue, which both consumer warpgroups of a CTA run on the same tile while the tensor pipe idles.  Each CTA gets
// half the shared memory, which must hold kMinTwoCtaStages A stages on the per-tap path or two strip stages.
static int size_launch(ConvOp& op, int bn, int num_sms) {
  ConvTcParams& p = op.p;
  p.BN = bn;
  p.n_tiles_n = ceil_div((int)align_up(op.Co, 16), bn);
  p.total_tiles = p.B * p.tiles_x * p.tiles_y * p.n_tiles_n;
  p.fd_ntn = make_fastdiv((unsigned)p.n_tiles_n);
  p.a_stage_bytes = kTileM * kKStage * 2;
  p.b_stage_bytes = (int)align_up(bn * kKStage * 2, 1024);
  p.bias_bytes = (int)align_up(p.n_tiles_n * bn * 4, 128);
  const int misc = 1024 /*barriers*/ + p.bias_bytes + 1024 /*alignment slack*/;
  const int b_resident_bytes = (int)align_up(p.n_chunks * bn * p.kc * 2, 1024);
  int grid = p.total_tiles < num_sms ? p.total_tiles : num_sms;
  const int grid_resident = grid / p.n_tiles_n * p.n_tiles_n;
  p.resident = op.reuse && grid_resident > 0 && b_resident_bytes <= kResidentPackLimit;
  p.strip = p.strip_w = p.strip_box_bytes = p.strip_sub_bytes = 0;
  if (p.resident && op.k == 3 && op.stride == 1 && p.tw >= 64 && p.cblocks <= kMaxStripBlocks && p.tw + 2 * op.dil <= 256) {
    p.strip_w = p.tw + 2 * op.dil;
    p.strip_box_bytes = p.strip_w * p.th * p.kc * 2;
    p.strip_sub_bytes = (int)align_up(p.strip_box_bytes, 1024);
    p.strip = (kSmemBudget - misc - b_resident_bytes) / (p.cblocks * p.strip_sub_bytes) >= 2;
  }
  if (p.strip) p.a_stage_bytes = p.cblocks * p.strip_sub_bytes;
  op.ctas_per_sm = p.resident && bn <= kTwoCtaMaxBN && p.total_tiles > num_sms &&
                           (kSmemBudgetTwoCtas - misc - b_resident_bytes) / p.a_stage_bytes >= (p.strip ? 2 : kMinTwoCtaStages)
                       ? 2
                       : 1;
  const int smem_budget = op.ctas_per_sm == 2 ? kSmemBudgetTwoCtas : kSmemBudget;
  int S;
  if (p.resident) {
    grid = op.ctas_per_sm == 2 ? (p.total_tiles < 2 * num_sms ? p.total_tiles : 2 * num_sms) / p.n_tiles_n * p.n_tiles_n : grid_resident;
    p.b_stage_bytes = 0;
    S = (smem_budget - misc - b_resident_bytes) / p.a_stage_bytes;
    p.b_bytes = b_resident_bytes;
  } else {
    S = (kSmemBudget - misc) / (p.a_stage_bytes + p.b_stage_bytes);
  }
  if (S > kMaxStages) S = kMaxStages;
  p.num_stages = S;
  if (!p.resident) p.b_bytes = S * p.b_stage_bytes;
  op.smem = S * p.a_stage_bytes + p.b_bytes + misc;
  op.grid = grid;
  return op.ctas_per_sm;
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
  p.kc = op.Ci_pad % 64 == 0 ? 64 : (op.Ci_pad % 32 == 0 ? 32 : 16);
  p.cblocks = op.Ci_pad / p.kc;
  p.taps = op.k * op.k;
  p.n_chunks = p.taps * p.cblocks;
  p.n_kstages = ceil_div(p.n_chunks, kKStage / p.kc);
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
  p.fd_tpi = make_fastdiv((unsigned)(p.tiles_x * p.tiles_y));
  p.fd_tx = make_fastdiv((unsigned)p.tiles_x);
  p.dil = op.dil;
  // N tile: whole Co if it fits in 128, else the largest multiple of 16 <= 128 dividing Co16 (Co_pad sized by the caller).  A layer
  // that this tile keeps at one CTA per SM takes BN = 64 instead when that admits the second CTA: each CTA then keeps half the pack and
  // A is read once per N tile (the second read from L2).  Outputs do not depend on BN: every output's K order is the same, and the
  // SiLU variant follows the channel mod 16, which n0 (a multiple of 16) leaves unchanged.
  const int co16 = (int)align_up(op.Co, 16);
  int bn = co16 <= 128 ? co16 : 128;
  if (co16 > 128 && co16 % 128 != 0) {
    for (int b = 128; b >= 16; b -= 16)
      if (co16 % b == 0) { bn = b; break; }
  }
  if (size_launch(op, bn, num_sms) == 1 && bn > kTwoCtaMaxBN && co16 % kTwoCtaMaxBN == 0 && size_launch(op, kTwoCtaMaxBN, num_sms) == 1)
    size_launch(op, bn, num_sms);
  MYOLO_REQUIRE(op.Co_pad >= p.n_tiles_n * p.BN, "conv_tc: Co_pad %d < %d", op.Co_pad, p.n_tiles_n * p.BN);
  MYOLO_REQUIRE(p.num_stages >= 2, "conv_tc: not enough shared memory for 2 stages");
  MYOLO_REQUIRE(p.n_tiles_n * p.BN * 4 <= kMaxBiasBytes, "conv_tc: %d output channels exceed the shared-memory bias buffer", p.n_tiles_n * p.BN);

  // ---- tensor maps ----
  const int esz = 2;
  const int sw = p.kc * 2;
  const TensorView& in = op.in;
  if (op.stride == 1) {
    uint64_t dims[4] = {(uint64_t)in.C, (uint64_t)in.W, (uint64_t)in.H, (uint64_t)in.B};
    uint64_t str[3] = {(uint64_t)in.ctot * esz, (uint64_t)in.W * in.ctot * esz, (uint64_t)in.H * in.W * in.ctot * esz};
    uint32_t box[4] = {(uint32_t)p.kc, (uint32_t)(p.strip ? p.strip_w : p.tw), (uint32_t)p.th, 1};
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

template <int KC, int BN, bool RES, int CTAS_PER_SM>
static cudaError_t launch_kernel(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(conv_tc_kernel<KC, BN, RES, CTAS_PER_SM>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBudget);
    if (e == cudaSuccess && CTAS_PER_SM == 2)   // two CTAs need the whole 228 KB carve-out, not whatever the driver would pick
      e = cudaFuncSetAttribute(conv_tc_kernel<KC, BN, RES, CTAS_PER_SM>, cudaFuncAttributePreferredSharedMemoryCarveout,
                               cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  return cudaLaunchKernelEx(&cfg, conv_tc_kernel<KC, BN, RES, CTAS_PER_SM>, op.tmA[0], op.tmA[1], op.tmA[2], op.tmA[3], op.tmB, op.p);
}

template <int KC, int BN, bool RES>
static cudaError_t launch_bn(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  if constexpr (BN <= kTwoCtaMaxBN)
    if (op.ctas_per_sm == 2) return launch_kernel<KC, BN, RES, 2>(op, cfg);
  if (op.ctas_per_sm != 1) return cudaErrorInvalidValue;
  return launch_kernel<KC, BN, RES, 1>(op, cfg);
}

template <int KC, bool RES>
static cudaError_t launch_kc(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  switch (op.p.BN) {
    case 16: return launch_bn<KC, 16, RES>(op, cfg);
    case 32: return launch_bn<KC, 32, RES>(op, cfg);
    case 48: return launch_bn<KC, 48, RES>(op, cfg);
    case 64: return launch_bn<KC, 64, RES>(op, cfg);
    case 80: return launch_bn<KC, 80, RES>(op, cfg);
    case 96: return launch_bn<KC, 96, RES>(op, cfg);
    case 112: return launch_bn<KC, 112, RES>(op, cfg);
    case 128: return launch_bn<KC, 128, RES>(op, cfg);
  }
  return cudaErrorInvalidValue;
}

template <bool RES>
static cudaError_t launch_res(const ConvOp& op, const cudaLaunchConfig_t& cfg) {
  switch (op.p.kc) {
    case 16: return launch_kc<16, RES>(op, cfg);
    case 32: return launch_kc<32, RES>(op, cfg);
    case 64: return launch_kc<64, RES>(op, cfg);
  }
  return cudaErrorInvalidValue;
}

int conv_tc_launch(const ConvOp& op, cudaStream_t stream) {
  MYOLO_REQUIRE(op.p.BN % 16 == 0 && op.p.BN >= 16 && op.p.BN <= 128, "conv_tc: unsupported N tile %d", op.p.BN);
  MYOLO_REQUIRE(op.p.kc == 16 || op.p.kc == 32 || op.p.kc == 64, "conv_tc: unsupported K chunk %d", op.p.kc);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(op.grid);
  cfg.blockDim = dim3(kNumThreads);
  cfg.dynamicSmemBytes = op.smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  MYOLO_CHECK_CUDA(op.p.residual != nullptr ? launch_res<true>(op, cfg) : launch_res<false>(op, cfg));
  g_launch_count++;
  return 0;
}

}  // namespace myolo
