// The wgmma GEMM of this library: the linear layers of the DINOv2 ViT-L/14 forward (row a1 of SURVEY.md §8; the hub
// module the reference calls at ae_net.py:46 runs them as fp32 cuBLAS GEMMs) and, as implicit GEMMs, the convolutions
// of the IST trunk (row a6, ist_trunk.cu; cuDNN in the reference).
//
// C[M,N] = A[M,K] . W[N,K]^T with both operands stored as bf16 hi/lo planes (x = hi + lo to ~2^-17) and accumulated
// as hi*hi + hi*lo + lo*hi in fp32 register accumulators -- the same fp32-faithful split as the similarity kernel
// (`passes = 1` = plain bf16).  Persistent CTAs, one 128 x bn output tile at a time:
//   warps 0-3   producer warpgroup (setmaxnreg down to 40): lane 0 of warp 0 issues the TMA loads (32-column k-blocks,
//               SWIZZLE_64B; A rows = 2-D boxes, or 4-D boxes of an NHWC plane when the GEMM is a convolution: one box
//               per filter tap and 32-channel block, zero fill = padding)
//   warps 4-11  two consumer warpgroups (setmaxnreg up to 232): wgmma m64 x bn x k16 on rows [0,64) / [64,128) of the
//               tile, then the epilogue straight from the accumulator fragments (fused bias / GELU / ReLU / LayerScale +
//               residual / shortcut / positional table -> fp32 rows or bf16 hi/lo planes for the next layer).  Each warp
//               handles its own 16 rows in 32-column chunks through a private staging buffer, so that every global
//               access is a run of whole 32-byte sectors; residual inputs of a chunk are loaded one chunk ahead.
// The epilogue never touches the operand ring: the producer streams the next tile's k-blocks while it runs.
// Two instantiation families: <swap=0> activation rows x output features; <swap=1> filters as the 128-row operand
// against 256 output pixels (the 128-channel convolutions).
#include "gigapose_kernels.h"
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace gp {

namespace {

constexpr int kBlockK = 32;
constexpr int kRowBytes = kBlockK * 2;            // 64 B rows, SWIZZLE_64B
constexpr int kStages = 4;                        // 48 KB stages
constexpr int kBM = 128, kBN = 256;
constexpr int kAPlane = kBM * kRowBytes;          // 8 KB
constexpr int kWPlane = kBN * kRowBytes;          // 16 KB
constexpr int kStageBytes = 2 * kAPlane + 2 * kWPlane;   // 48 KB
constexpr int kEpiWarps = 8;
constexpr int kThreads = 4 * 32 + kEpiWarps * 32;
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
static_assert(128 * kProducerRegs + kEpiWarps * 32 * kConsumerRegs <= 65536, "register file");
// Per-warp staging of one 32-column chunk of the warp's 16 rows.  Row pitches keep the fragment-layout accesses free
// of bank conflicts: bf16 planes 144 B (hi 64 B | lo 64 B | pad), fp32 rows 160 B (128 B | pad); the swapped form
// holds 32 pixel rows of 80 B (16 channels hi 32 B | lo 32 B | pad).
constexpr int kStagePitchPlanes = 144, kStagePitchF32 = 160, kStagePitchSwap = 80;
constexpr int kStageBufBytes = 16 * kStagePitchF32;
static_assert(16 * kStagePitchPlanes <= kStageBufBytes && 32 * kStagePitchSwap <= kStageBufBytes, "staging buffer");

struct __align__(8) GemmSmemTail {
  float bias_s[2][kBN];                           // per-tile bias / LayerScale columns, indexed by tile parity
  float gamma_s[2][kBN];
  uint8_t stage_buf[kEpiWarps][kStageBufBytes];
  uint64_t full_bar[kStages];
  uint64_t empty_bar[kStages];
};
constexpr int kSmemBytes = 1024 + kStages * kStageBytes + sizeof(GemmSmemTail);

// Grouped rasterisation: 16 m-tiles x all n-tiles per group, m fastest inside a group.  With plain m-fastest order all
// CTAs stream the same 256-row weight tile at the same moment and serialise on its L2 lines; in a group every
// weight tile is shared by <= 16 CTAs and every activation tile by <= num_n CTAs.
constexpr int kGroupM = 16;
__device__ __forceinline__ void tile_coords(int tile, int num_m, int num_n, int& m_tile, int& n_tile) {
  const int per_group = kGroupM * num_n;
  const int g = tile / per_group, idx = tile - g * per_group;
  const int m_first = g * kGroupM;
  const int gm = min(kGroupM, num_m - m_first);
  n_tile = idx / gm;
  m_tile = m_first + (idx - n_tile * gm);
}

// GELU(x) = 0.5 x (1 + erf(x / sqrt 2)) through erfc(u) = t (a1 + t (a2 + t (a3 + t (a4 + t a5)))) exp(-u^2), t = 1 / (1 + p u)
// (Abramowitz & Stegun 7.1.26, |error| <= 1.5e-7 on erf): 1 + erf = erfc(|u|) for x < 0 (no cancellation) and 2 - erfc(|u|)
// otherwise.  14 instructions per element instead of erff's 25 (fc1 was the one layer whose epilogue was slower than its
// MMAs); against the exact function the result is off by <= 4.2e-7 absolute over [-8, 8] -- the same as the fp32 erff form
// (4.5e-7: both are dominated by the fp32 rounding of the final products).
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float t, e;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.231641888f, ax, 1.0f)));          // p / sqrt(2), p = 0.3275911
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * x * -0.72134752f));                   // exp(-x^2 / 2)
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  const float q = poly * t * e;                                                              // erfc(|x| / sqrt 2)
  return 0.5f * x * (x < 0.f ? q : 2.0f - q);
}

__device__ __forceinline__ uint32_t pack_bf16(__nv_bfloat16 a, __nv_bfloat16 b) {
  return (uint32_t)__bfloat16_as_ushort(a) | ((uint32_t)__bfloat16_as_ushort(b) << 16);
}

}  // namespace

// cycle stamps of CTA 0 of a launch with GemmParams::stamp set (diagnostics: gp_debug_gemm_timeline), for the CTA's
// first kStampTiles tiles: [4 * tile + {0: MMA start, 1: MMA done, 2: epilogue start, 3: epilogue end}],
// [63] = kernel start, [64 + tile] = the tile's first k-block has landed (first full barrier passed)
constexpr int kStampTiles = 15;
__device__ long long g_gemm_stamp[128];
#define GSTAMP(i) do { if (blockIdx.x == 0 && p.stamp) g_gemm_stamp[i] = clock64(); } while (0)

// One k-block (32 columns of K, up to 3 split passes) of a consumer warpgroup's 64 x kN accumulator.
template <int kN, bool kF16>
__device__ __forceinline__ void gemm_kblock(float (&d)[kN / 2], uint32_t a_hi, uint32_t a_lo, uint32_t w_hi, uint32_t w_lo,
                                            int passes, bool first) {
#pragma unroll
  for (int pass = 0; pass < 3; ++pass) {
    if (pass < passes) {
      const uint32_t a = (pass == 2 ? a_lo : a_hi), w = (pass == 1 ? w_lo : w_hi);
#pragma unroll
      for (int k16 = 0; k16 < kBlockK / 16; ++k16) {
        const uint64_t da = wgmma_desc_kmajor<kRowBytes>(a + k16 * 32), dw = wgmma_desc_kmajor<kRowBytes>(w + k16 * 32);
        const uint32_t accum = (!first || pass != 0 || k16 != 0) ? 1u : 0u;
        if constexpr (kN == 256) { if constexpr (kF16) wgmma_ss_n256_f16(d, da, dw, accum); else wgmma_ss_n256_bf16(d, da, dw, accum); }
        if constexpr (kN == 192) { if constexpr (kF16) wgmma_ss_n192_f16(d, da, dw, accum); else wgmma_ss_n192_bf16(d, da, dw, accum); }
      }
    }
  }
}

// kMode (GemmMode) is a template parameter: every layer type gets its own epilogue without the other modes' predicated
// code and registers.
// kSwap = false: rows of C are activation rows (tokens / output pixels), columns are output features.
// kSwap = true (convolutions with 128 output channels): the roles are exchanged -- the 128-row operand is the filter
// bank [128, K] and the 256-row operand is a tile of 256 output pixels, so that the tensor pipe still runs N = 256
// instructions (an N = 128 instruction re-reads its A operand from shared memory twice as often per FLOP); the epilogue
// transposes the [channel, pixel] accumulator back to NHWC.
// kTileN (192 / 256 output columns per tile) and kF16 (operand planes hold fp16 instead of bf16 pairs) are
// template parameters too: a runtime choice inside the k-loop makes ptxas insert warpgroup waits between the MMAs.
template <bool kSwap, int kTileN, bool kF16, int kMode>
__global__ void __launch_bounds__(kThreads, 1)
vit_gemm_kernel(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
                const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo, GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  pdl_trigger();                                     // the next kernel's CTAs may take SMs as this grid's CTAs retire
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  GemmSmemTail& tail = *reinterpret_cast<GemmSmemTail*>(smem + kStages * kStageBytes);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int passes = p.passes;
  constexpr int bn = kTileN;
  const int M_rows = p.m_dev ? min(*p.m_dev, p.M) : p.M;    // data-dependent row count (IST regressor): read on the device
  const int num_m = (M_rows + kBM - 1) / kBM, num_n = p.N / bn;
  const int num_tiles = num_m * num_n;
  const int num_kb = p.K / kBlockK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&tail.full_bar[s], 1); mbar_init(&tail.empty_bar[s], kEpiWarps); }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_w_hi);
    if (passes == 3) { tma_prefetch_desc(&tm_a_lo); tma_prefetch_desc(&tm_w_lo); }
  }
  __syncthreads();
  pdl_wait();                                        // everything above overlapped the previous kernel's tail
  if (threadIdx.x == 0) GSTAMP(63);

  if (warp < 4) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == 0 && lane == 0) {
      int stage = 0; uint32_t phase = 0;
      const uint32_t tx = (passes == 3 ? 2 : 1) * (kAPlane + bn * kRowBytes);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
        int mt, nt;
        tile_coords(tile, num_m, num_n, mt, nt);
        const int m0 = mt * kBM, n0 = nt * bn;
        int img = 0, y0 = 0;
        if (p.conv) { const int hw = p.Ho * p.Wo, pix0 = kSwap ? n0 : m0; img = pix0 / hw; y0 = (pix0 - img * hw) / p.Wo; }
        for (int kb = 0; kb < num_kb; ++kb) {
          mbar_wait(&tail.empty_bar[stage], phase ^ 1);
          uint8_t* st = smem + stage * kStageBytes;
          mbar_arrive_expect_tx(&tail.full_bar[stage], tx);
          // the pixel operand (A, or W when kSwap) of a convolution: k-block = (tap ky,kx ; 32-channel block cb), a
          // shifted, strided window of the NHWC plane; the other operand is a plain [rows, K] matrix
          int cb = 0, cx = 0, cy = 0;
          if (p.conv) {
            const int tap = kb / p.cblocks;
            cb = kb - tap * p.cblocks;
            const int ky = tap / p.kw, kx = tap - ky * p.kw;
            cx = kx - p.pad; cy = y0 * p.stride + ky - p.pad;
          }
          auto load2 = [&](void* dst, const CUtensorMap* map, int c0, int c1) { tma_load_2d(dst, map, &tail.full_bar[stage], c0, c1); };
          auto load4 = [&](void* dst, const CUtensorMap* map) {
            tma_load_4d(dst, map, &tail.full_bar[stage], cb * kBlockK, cx, cy, img);
          };
          if (p.conv && !kSwap) {
            load4(st, &tm_a_hi);
            if (passes == 3) load4(st + kAPlane, &tm_a_lo);
          } else {
            load2(st, &tm_a_hi, kb * kBlockK, m0);
            if (passes == 3) load2(st + kAPlane, &tm_a_lo, kb * kBlockK, m0);
          }
          if (p.conv && kSwap) {
            load4(st + 2 * kAPlane, &tm_w_hi);
            if (passes == 3) load4(st + 2 * kAPlane + kWPlane, &tm_w_lo);
          } else {
            load2(st + 2 * kAPlane, &tm_w_hi, kb * kBlockK, n0);
            if (passes == 3) load2(st + 2 * kAPlane + kWPlane, &tm_w_lo, kb * kBlockK, n0);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    setmaxnreg_inc<kConsumerRegs>();
    const int e = warp - 4, etid = e * 32 + lane;
    const int wg = e >> 2, wl = e & 3;                 // warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    const int wrow0 = wg * 64 + wl * 16;               // this warp's 16 rows of the tile (MMA fragments and epilogue)
    const int fr = lane >> 2, fc = 2 * (lane & 3);     // fragment: rows wrow0 + fr (+ 8), columns 8 j + fc (+ 1)
    constexpr bool kPlanesOut = kMode == GEMM_PLANES || kMode == GEMM_PLANES_GELU || kMode == GEMM_QKV_HEADS ||
                                kMode == GEMM_PLANES_RELU || kMode == GEMM_PLANES_ADD_RELU;
    constexpr bool kResIn = kMode == GEMM_SCALE_RESIDUAL || kMode == GEMM_PLANES_ADD_RELU;
    constexpr int kChunks = kTileN / 32;
    uint8_t* stg = tail.stage_buf[e];
    int stage = 0; uint32_t phase = 0, unit = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++unit) {
      const uint32_t acc_i = unit & 1u;
      const bool stamp = e == 0 && lane == 0 && unit < kStampTiles;
      int mt, nt;
      tile_coords(tile, num_m, num_n, mt, nt);
      const int m0 = mt * kBM, ntile0 = nt * bn;
      if (stamp) GSTAMP(unit * 4 + 0);
      // per-column vectors (or, swapped, the bias of the fragment's two channel rows): loaded now, used after the MMAs
      float bias_v = 0.f, gamma_v = 0.f, bias_r[2] = {0.f, 0.f};
      if (!kSwap && etid < bn) {
        bias_v = __ldg(p.bias + ntile0 + etid);
        if (kMode == GEMM_SCALE_RESIDUAL) gamma_v = __ldg(p.gamma + ntile0 + etid);
      }
      if (kSwap) { bias_r[0] = __ldg(p.bias + m0 + wrow0 + fr); bias_r[1] = __ldg(p.bias + m0 + wrow0 + fr + 8); }

      // The four 16-byte pieces this lane moves between the staging buffer and global memory in every chunk.
      // Row-major forms: piece k is in row 4 k + lane / 8 of the warp's 16; bf16 planes: lanes 0-3 / 4-7 of a row take
      // the hi / lo plane, 64 B each; fp32: 8 lanes x 16 B = 128 B.  Swapped form: pixel 8 k + lane / 4 of the chunk's
      // 32, lanes 0-1 / 2-3 take the 32 bytes (16 channels) of the hi / lo plane.
      size_t row_off[4];                               // element offset of the piece's output row (row-major forms)
      uint32_t row_ok = 0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        row_off[k] = 0;
        if constexpr (!kSwap) {
          const int m = m0 + wrow0 + 4 * k + (lane >> 3);
          if (m < M_rows) row_ok |= 1u << k;
          if (kMode == GEMM_QKV_HEADS) {               // head-major: [q|k|v][crop][head][token][64]
            const int img = m / p.tokens_per_img, tok = m - img * p.tokens_per_img;
            row_off[k] = ((size_t)img * 16 * p.tokens_per_img + tok) * 64;
          } else if (kMode == GEMM_PATCH_EMBED) {      // patch row -> token row (CLS first)
            const int img = m / p.patches_per_img, pp = m - img * p.patches_per_img;
            row_off[k] = ((size_t)img * p.tokens_per_img + 1 + pp) * p.N;
          } else {
            row_off[k] = (size_t)m * p.N;
          }
        } else {
          row_ok |= 1u << k;                           // swap: M % 128 == 0 and N % 256 == 0, no partial tiles
        }
      }
      auto piece_smem = [&](int k) -> uint8_t* {
        if constexpr (kSwap) return stg + (8 * k + (lane >> 2)) * kStagePitchSwap + (lane & 3) * 16;
        else if constexpr (kPlanesOut) return stg + (4 * k + (lane >> 3)) * kStagePitchPlanes + (lane & 7) * 16;
        else return stg + (4 * k + (lane >> 3)) * kStagePitchF32 + (lane & 7) * 16;
      };
      // byte address of piece k of chunk c in the fp32 rows `x` or in the plane pair (hi, lo)
      auto piece_gmem = [&](int k, int c, const void* x, const void* hi, const void* lo) -> const uint8_t* {
        if constexpr (kSwap) {
          const size_t pix = (size_t)ntile0 + c * 32 + 8 * k + (lane >> 2);
          const void* plane = (lane & 2) ? lo : hi;
          return reinterpret_cast<const uint8_t*>(plane) + (pix * p.M + m0 + wrow0) * 2 + (lane & 1) * 16;
        } else {
          const int n = ntile0 + c * 32;
          size_t col = (size_t)n;
          if (kMode == GEMM_QKV_HEADS) {
            const int which = n >> 10, head = (n & 1023) >> 6;
            col = ((size_t)which * p.qkv_crop_stride * 16 + head) * p.tokens_per_img * 64 + (n & 63);
          }
          if constexpr (kPlanesOut) {
            const void* plane = (lane & 4) ? lo : hi;
            return reinterpret_cast<const uint8_t*>(plane) + (row_off[k] + col) * 2 + (lane & 3) * 16;
          } else {
            return reinterpret_cast<const uint8_t*>(x) + (row_off[k] + col) * 4 + (lane & 7) * 16;
          }
        }
      };
      // residual inputs (x += ... / the shortcut planes) of a chunk, one chunk ahead of its use
      uint4 res[4];
      auto load_res = [&](int c) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          res[k] = make_uint4(0, 0, 0, 0);
          if ((row_ok >> k) & 1u) res[k] = *reinterpret_cast<const uint4*>(piece_gmem(k, c, p.x, p.res_hi, p.res_lo));
        }
      };
      // patch embedding: the positional-table rows of the fragment's two rows
      const float* pos_row[2] = {nullptr, nullptr};
      bool frag_row_ok[2] = {false, false};
      if (kMode == GEMM_PATCH_EMBED) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m = m0 + wrow0 + fr + 8 * h;
          const int img = m / p.patches_per_img, pp = m - img * p.patches_per_img;
          pos_row[h] = p.pos + (size_t)(1 + pp) * p.N;
          frag_row_ok[h] = m < M_rows;
        }
      }

      // ---------------- main loop: wgmma from the operand ring into registers
      float frag[kTileN / 2];
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&tail.full_bar[stage], phase);
        if (kb == 0 && stamp) GSTAMP(64 + unit);
        const uint32_t st = smem_u32(smem + stage * kStageBytes);
        const uint32_t a_hi = st + wg * (kAPlane / 2), a_lo = a_hi + kAPlane;
        const uint32_t w_hi = st + 2 * kAPlane, w_lo = w_hi + kWPlane;
        acc_fence(frag);
        wgmma_fence();
        gemm_kblock<kTileN, kF16>(frag, a_hi, a_lo, w_hi, w_lo, passes, kb == 0);
        wgmma_commit();
        wgmma_wait<1>();                               // the previous k-block's MMAs have retired: its stage is free
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&tail.empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == kStages) { stage = 0; phase ^= 1; }
      }
      if (kResIn) load_res(0);                         // in flight while the last k-block's MMAs retire
      wgmma_wait<0>();
      acc_fence(frag);
      if (lane == 0) mbar_arrive(&tail.empty_bar[prev_stage]);
      if (stamp) GSTAMP(unit * 4 + 1);
      if (!kSwap && etid < bn) {
        tail.bias_s[acc_i][etid] = bias_v;
        if (kMode == GEMM_SCALE_RESIDUAL) tail.gamma_s[acc_i][etid] = gamma_v;
      }
      // the vectors are visible to both warpgroups; since every warp has passed this barrier, none still reads the
      // other parity's vectors of the tile before
      named_barrier_sync(1, kEpiWarps * 32);
      if (stamp) GSTAMP(unit * 4 + 2);

      // ---------------- epilogue, 32 columns at a time: residual in -> fragment math -> staging -> global
      const float* sb = tail.bias_s[acc_i];
      const float* sg = tail.gamma_s[acc_i];
#pragma unroll
      for (int c = 0; c < kChunks; ++c) {
        if (kResIn) {
#pragma unroll
          for (int k = 0; k < 4; ++k) *reinterpret_cast<uint4*>(piece_smem(k)) = res[k];
          if (c + 1 < kChunks) load_res(c + 1);
          __syncwarp();
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int j8 = c * 4 + jj;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const float a0 = frag[4 * j8 + 2 * h], a1 = frag[4 * j8 + 2 * h + 1];
            const int rr = fr + 8 * h;                 // row of the warp's 16
            if constexpr (kSwap) {
              // thread = output channels rr, columns = pixels: the values land in their NHWC pixel rows
              float v[2] = {a0 + bias_r[h], a1 + bias_r[h]};
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                uint8_t* px = stg + (jj * 8 + fc + i) * kStagePitchSwap + rr * 2;
                if (kMode == GEMM_PLANES_ADD_RELU) {
                  v[i] += __uint_as_float((uint32_t)*reinterpret_cast<const uint16_t*>(px) << 16);
                  v[i] += __uint_as_float((uint32_t)*reinterpret_cast<const uint16_t*>(px + 32) << 16);
                }
                if (kMode == GEMM_PLANES_RELU || kMode == GEMM_PLANES_ADD_RELU) v[i] = fmaxf(v[i], 0.f);
                const __nv_bfloat16 hb = __float2bfloat16_rn(v[i]);
                *reinterpret_cast<uint16_t*>(px) = __bfloat16_as_ushort(hb);
                *reinterpret_cast<uint16_t*>(px + 32) = __bfloat16_as_ushort(__float2bfloat16_rn(v[i] - __bfloat162float(hb)));
              }
            } else {
              const int col = c * 32 + jj * 8 + fc;    // column of the tile
              const float2 bb = *reinterpret_cast<const float2*>(sb + col);
              float v0 = (p.acc_scale != 0.f ? a0 * p.acc_scale : a0) + bb.x;
              float v1 = (p.acc_scale != 0.f ? a1 * p.acc_scale : a1) + bb.y;
              if constexpr (kPlanesOut) {
                uint32_t* w_hi = reinterpret_cast<uint32_t*>(stg + rr * kStagePitchPlanes + (jj * 8 + fc) * 2);
                uint32_t* w_lo = w_hi + 16;
                if (kMode == GEMM_PLANES_ADD_RELU) {   // BasicBlock: relu(shortcut + bn2(conv2(.)))   (resnet.py:45-50)
                  const uint32_t rh = *w_hi, rl = *w_lo;
                  v0 += __uint_as_float(rh << 16) + __uint_as_float(rl << 16);
                  v1 += __uint_as_float(rh & 0xffff0000u) + __uint_as_float(rl & 0xffff0000u);
                }
                if (kMode == GEMM_PLANES_GELU) { v0 = gelu_erf(v0); v1 = gelu_erf(v1); }
                if (kMode == GEMM_PLANES_RELU || kMode == GEMM_PLANES_ADD_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if constexpr (kF16) {                  // saturating: a value beyond the fp16 range stays finite (and wrong) instead of inf
                  v0 = fminf(fmaxf(v0, -65504.f), 65504.f);
                  v1 = fminf(fmaxf(v1, -65504.f), 65504.f);
                  const __half ah = __float2half_rn(v0), bh = __float2half_rn(v1);
                  *w_hi = (uint32_t)__half_as_ushort(ah) | ((uint32_t)__half_as_ushort(bh) << 16);
                  *w_lo = (uint32_t)__half_as_ushort(__float2half_rn(v0 - __half2float(ah))) |
                          ((uint32_t)__half_as_ushort(__float2half_rn(v1 - __half2float(bh))) << 16);
                } else {
                  const __nv_bfloat16 ah = __float2bfloat16_rn(v0), bh = __float2bfloat16_rn(v1);
                  *w_hi = pack_bf16(ah, bh);
                  *w_lo = pack_bf16(__float2bfloat16_rn(v0 - __bfloat162float(ah)), __float2bfloat16_rn(v1 - __bfloat162float(bh)));
                }
              } else {
                float2* w = reinterpret_cast<float2*>(stg + rr * kStagePitchF32 + (jj * 8 + fc) * 4);
                float2 o;
                if (kMode == GEMM_SCALE_RESIDUAL) {    // x += gamma * (acc + bias)   (blocks: ls1 / ls2 + residual)
                  const float2 g = *reinterpret_cast<const float2*>(sg + col), xv = *w;
                  o = make_float2(xv.x + g.x * v0, xv.y + g.y * v1);
                } else if (kMode == GEMM_ROWS_F32 || kMode == GEMM_ROWS_F32_RELU) {   // plain fp32 rows (last 1x1
                  const float floor_v = kMode == GEMM_ROWS_F32_RELU ? 0.f : -INFINITY;  // convolution of the IST trunk;
                  o = make_float2(fmaxf(v0, floor_v), fmaxf(v1, floor_v));            // second hidden layer of the IST MLP)
                } else {                               // GEMM_PATCH_EMBED: + positional table
                  const int n = ntile0 + col;
                  o = make_float2(v0 + (frag_row_ok[h] ? __ldg(pos_row[h] + n) : 0.f),
                                  v1 + (frag_row_ok[h] ? __ldg(pos_row[h] + n + 1) : 0.f));
                }
                *w = o;
              }
            }
          }
        }
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 4; ++k)
          if ((row_ok >> k) & 1u)
            *reinterpret_cast<uint4*>(const_cast<uint8_t*>(piece_gmem(k, c, p.x, p.out_hi, p.out_lo))) =
                *reinterpret_cast<const uint4*>(piece_smem(k));
        __syncwarp();                                  // the staging buffer is free for the next chunk
      }
      if (stamp) GSTAMP(unit * 4 + 3);
    }
  }
}

cudaError_t read_gemm_stamps(long long* host128) { return cudaMemcpyFromSymbol(host128, g_gemm_stamp, sizeof(g_gemm_stamp)); }

namespace {
template <bool kSwap, int kTileN, bool kF16, int kMode>
cudaError_t launch_mode(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi, const CUtensorMap& w_lo,
                        const GemmParams& p, int grid, cudaStream_t stream) {
  return launch_ex(vit_gemm_kernel<kSwap, kTileN, kF16, kMode>, dim3(grid), dim3(kThreads), kSmemBytes, stream, 1, true, a_hi,
                   a_lo, w_hi, w_lo, p);
}
}  // namespace

// Instantiated combinations: every mode at 256 columns (bf16); the three bf16-plane modes also at 192 columns and with
// the filters as the 128-row operand (kSwap, 256 columns); fp16 pairs for the two regressor layers.
bool gemm_config_supported(const GemmParams& p, const char** why) {
  if (why) *why = nullptr;
  auto no = [&](const char* msg) { if (why) *why = msg; return false; };
  const int bn = p.bn > 0 ? p.bn : kBN;
  const bool plane_mode = p.mode == GEMM_PLANES || p.mode == GEMM_PLANES_RELU || p.mode == GEMM_PLANES_ADD_RELU;
  if (bn != 192 && bn != 256) return no("bn must be 192 or 256 (0 = 256)");
  if (p.N <= 0 || p.N % bn != 0) return no("N must be a positive multiple of bn");
  if (p.K <= 0 || p.K % kBlockK != 0) return no("K must be a positive multiple of 32");
  if (p.passes != 1 && p.passes != 3) return no("passes must be 1 or 3");
  if (p.mode < GEMM_PLANES || p.mode > GEMM_ROWS_F32_RELU) return no("unknown mode");
  const int tile_pixels = p.swap ? bn : kBM;
  if (p.conv && (p.Wo <= 0 || tile_pixels % p.Wo != 0 || p.M % kBM != 0 || p.cblocks <= 0))
    return no("convolution geometry does not tile");
  if (p.swap && (bn != kBN || p.M % kBM != 0 || p.f16 || !plane_mode))
    return no("swap needs bn = 256, M % 128 == 0, bf16 planes and a plane mode without GELU");
  if (p.f16 && (bn != kBN || (p.mode != GEMM_PLANES_RELU && p.mode != GEMM_ROWS_F32_RELU)))
    return no("f16 needs bn = 256 and mode PLANES_RELU or ROWS_F32_RELU");
  if (bn == 192 && !plane_mode) return no("bn = 192 supports the modes PLANES, PLANES_RELU and PLANES_ADD_RELU only");
  return true;
}

// Anything gemm_config_supported() rejects returns cudaErrorInvalidValue.
cudaError_t launch_vit_gemm(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi,
                            const CUtensorMap& w_lo, const GemmParams& p, int num_sms, cudaStream_t stream) {
  if (p.M <= 0) return cudaSuccess;
  if (!gemm_config_supported(p)) return cudaErrorInvalidValue;
  const int bn = p.bn > 0 ? p.bn : kBN;
  const int tiles = ((p.M + kBM - 1) / kBM) * (p.N / bn);
  const int grid = tiles < num_sms ? tiles : num_sms;
#define GP_GEMM_CASE(SWAP, N, F16, MODE) \
  case MODE: return launch_mode<SWAP, N, F16, MODE>(a_hi, a_lo, w_hi, w_lo, p, grid, stream);
#define GP_GEMM_PLANE_MODES(SWAP, N)            \
  switch (p.mode) {                             \
    GP_GEMM_CASE(SWAP, N, false, GEMM_PLANES)      \
    GP_GEMM_CASE(SWAP, N, false, GEMM_PLANES_RELU) \
    GP_GEMM_CASE(SWAP, N, false, GEMM_PLANES_ADD_RELU) \
    default: return cudaErrorInvalidValue;      \
  }
  if (p.swap) GP_GEMM_PLANE_MODES(true, 256)
  if (p.f16) {
    switch (p.mode) {
      GP_GEMM_CASE(false, 256, true, GEMM_PLANES_RELU)
      GP_GEMM_CASE(false, 256, true, GEMM_ROWS_F32_RELU)
      default: return cudaErrorInvalidValue;
    }
  }
  if (bn == 192) GP_GEMM_PLANE_MODES(false, 192)
  switch (p.mode) {
    GP_GEMM_CASE(false, 256, false, GEMM_PLANES)
    GP_GEMM_CASE(false, 256, false, GEMM_PLANES_GELU)
    GP_GEMM_CASE(false, 256, false, GEMM_SCALE_RESIDUAL)
    GP_GEMM_CASE(false, 256, false, GEMM_PATCH_EMBED)
    GP_GEMM_CASE(false, 256, false, GEMM_QKV_HEADS)
    GP_GEMM_CASE(false, 256, false, GEMM_PLANES_RELU)
    GP_GEMM_CASE(false, 256, false, GEMM_PLANES_ADD_RELU)
    GP_GEMM_CASE(false, 256, false, GEMM_ROWS_F32)
    GP_GEMM_CASE(false, 256, false, GEMM_ROWS_F32_RELU)
    default: return cudaErrorInvalidValue;
  }
#undef GP_GEMM_PLANE_MODES
#undef GP_GEMM_CASE
}

}  // namespace gp
