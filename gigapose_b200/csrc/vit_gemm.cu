// The wgmma GEMM of this library: the linear layers of the DINOv2 ViT-L/14 forward (row a1 of SURVEY.md §8; the hub
// module the reference calls at ae_net.py:46 runs them as fp32 cuBLAS GEMMs) and, as implicit GEMMs, the convolutions
// of the IST trunk (row a6, ist_trunk.cu; cuDNN in the reference).
//
// C[M,N] = A[M,K] . W[N,K]^T with both operands stored as bf16 hi/lo planes (x = hi + lo to ~2^-17) and accumulated
// as hi*hi + hi*lo + lo*hi in fp32 register accumulators -- the same fp32-faithful split as the similarity kernel
// (`passes = 1` = plain bf16).  Persistent CTAs, one 128 x bn output tile at a time:
//   warp 0      TMA producer   (32-column k-blocks, SWIZZLE_64B; A rows = 2-D boxes, or 4-D boxes of an NHWC plane when
//                              the GEMM is a convolution: one box per filter tap and 32-channel block, zero fill = padding)
//   warps 4-11  two consumer warpgroups: wgmma m64 x bn x k16 on rows [0,64) / [64,128) of the tile, then the epilogue
//               (the accumulator goes through shared memory so that a thread owns one row: fused bias / GELU / ReLU /
//               LayerScale + residual / shortcut / positional table -> fp32 rows or bf16 hi/lo planes for the next
//               layer; stores are transposed through shared memory into full 64-byte segments).
// The staged accumulator reuses the operand ring, so the producer starts the next tile's loads once the epilogue has
// read it.  Two instantiation families: <swap=0> activation rows x output features; <swap=1> filters as the 128-row
// operand against 256 output pixels (the 128-channel convolutions).
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
constexpr int kAccPitch = kBN + 4;                // fp32 words per staged accumulator row (+16 B: conflict-free float4 reads)
static_assert(kBM * kAccPitch * 4 <= kStages * kStageBytes, "the staged accumulator lives in the operand ring");

struct __align__(8) GemmSmemTail {
  float bias_s[2][kBN];                           // per-tile bias / LayerScale columns
  float gamma_s[2][kBN];
  uint8_t stage_buf[kEpiWarps][32 * 80];          // per-warp transposition buffer: 32 rows x (64 B + 16 B pad)
  uint64_t full_bar[kStages];
  uint64_t empty_bar[kStages];
  uint64_t ring_free_bar;                         // the epilogue has read the staged accumulator
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

// cycle stamps of CTA 0 for the QKV-shaped GEMM (diagnostics: gp_debug_gemm_timeline): [tile][0..3] =
// MMA start, MMA done, epilogue start, epilogue end; [63] = kernel start
__device__ long long g_gemm_stamp[64];
#define GSTAMP(i) do { if (blockIdx.x == 0 && p.N == 3072 && (i) < 64) g_gemm_stamp[i] = clock64(); } while (0)

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
  float* acc_s = reinterpret_cast<float*>(smem);     // [kBM][kAccPitch] staged accumulator (over the operand ring)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int passes = p.passes;
  constexpr int bn = kTileN;
  const int M_rows = p.m_dev ? min(*p.m_dev, p.M) : p.M;    // data-dependent row count (IST regressor): read on the device
  const int num_m = (M_rows + kBM - 1) / kBM, num_n = p.N / bn;
  const int num_tiles = num_m * num_n;
  const int num_kb = p.K / kBlockK;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&tail.full_bar[s], 1); mbar_init(&tail.empty_bar[s], kEpiWarps); }
    mbar_init(&tail.ring_free_bar, kEpiWarps);
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_a_hi); tma_prefetch_desc(&tm_w_hi);
    if (passes == 3) { tma_prefetch_desc(&tm_a_lo); tma_prefetch_desc(&tm_w_lo); }
  }
  __syncthreads();
  pdl_wait();                                        // everything above overlapped the previous kernel's tail
  if (threadIdx.x == 0) GSTAMP(63);

  if (warp == 0) {
    if (lane == 0) {
      int stage = 0; uint32_t phase = 0, unit = 0;
      const uint32_t tx = (passes == 3 ? 2 : 1) * (kAPlane + bn * kRowBytes);
      for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++unit) {
        int mt, nt;
        tile_coords(tile, num_m, num_n, mt, nt);
        const int m0 = mt * kBM, n0 = nt * bn;
        int img = 0, y0 = 0;
        if (p.conv) { const int hw = p.Ho * p.Wo, pix0 = kSwap ? n0 : m0; img = pix0 / hw; y0 = (pix0 - img * hw) / p.Wo; }
        if (unit > 0) mbar_wait(&tail.ring_free_bar, (unit - 1) & 1u);   // the previous tile's staged accumulator was read
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
  } else if (warp >= 4) {
    const int e = warp - 4, q = e & 3, ch = e >> 2;
    const int r = q * 32 + lane;                       // epilogue: this thread's row of the tile
    const int etid = e * 32 + lane;
    const int wg = e >> 2, wl = e & 3;                 // MMA: warpgroup wg owns tile rows [64 wg, 64 wg + 64)
    int stage = 0; uint32_t phase = 0, unit = 0;
    for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x, ++unit) {
      const uint32_t acc_i = unit & 1u;
      int mt, nt;
      tile_coords(tile, num_m, num_n, mt, nt);
      if (e == 0 && lane == 0) GSTAMP(unit * 4 + 0);
      // ---------------- main loop: wgmma from the operand ring into registers
      float frag[kTileN / 2];
      int prev_stage = -1;
      for (int kb = 0; kb < num_kb; ++kb) {
        mbar_wait(&tail.full_bar[stage], phase);
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
      wgmma_wait<0>();
      acc_fence(frag);
      if (lane == 0) mbar_arrive(&tail.empty_bar[prev_stage]);
      if (e == 0 && lane == 0) GSTAMP(unit * 4 + 1);
      // ---------------- stage the accumulator (row-major fp32) and the per-column vectors
      named_barrier_sync(1, kEpiWarps * 32);           // both warpgroups are done reading the ring
      {
        const int row0 = wg * 64 + wl * 16 + (lane >> 2), col0 = 2 * (lane & 3);
#pragma unroll
        for (int j8 = 0; j8 < kTileN / 8; ++j8) {
          {
            *reinterpret_cast<float2*>(acc_s + row0 * kAccPitch + j8 * 8 + col0) = make_float2(frag[4 * j8], frag[4 * j8 + 1]);
            *reinterpret_cast<float2*>(acc_s + (row0 + 8) * kAccPitch + j8 * 8 + col0) = make_float2(frag[4 * j8 + 2], frag[4 * j8 + 3]);
          }
        }
      }
      const int ntile0 = nt * bn;
      if (!kSwap && etid < bn) {
        tail.bias_s[acc_i][etid] = __ldg(p.bias + ntile0 + etid);
        if (kMode == GEMM_SCALE_RESIDUAL) tail.gamma_s[acc_i][etid] = __ldg(p.gamma + ntile0 + etid);
      }
      named_barrier_sync(1, kEpiWarps * 32);
      if (e == 0 && lane == 0) GSTAMP(unit * 4 + 2);
      // ---------------- epilogue: thread = row r, columns [ch * bn/2, (ch + 1) * bn/2) in chunks of 32
      const uint32_t acc = acc_i;
      const int m = mt * kBM + r;
      const int half_cols = bn >> 1;                   // columns per epilogue warp: 96 / 128
      const int n0 = ntile0 + ch * half_cols;
      const float* sb = tail.bias_s[acc] + ch * half_cols;
      const float* sg = tail.gamma_s[acc] + ch * half_cols;
      const bool row_ok = m < M_rows;
      size_t out_row = (size_t)m;
      const float* pos_row = nullptr;
      if (kMode == GEMM_PATCH_EMBED) {                // patch row -> token row (CLS first), + positional table
        const int img = m / p.patches_per_img, pp = m - img * p.patches_per_img;
        out_row = (size_t)img * p.tokens_per_img + 1 + pp;
        pos_row = p.pos + (size_t)(1 + pp) * p.N;
      }

      uint8_t* stg = tail.stage_buf[e];
      const unsigned okmask = __ballot_sync(0xffffffffu, row_ok);
      // One warp-wide store instruction of the natural "thread = row" mapping touches 32 different rows with 16 bytes
      // each (32 half-written sectors).  Rows are therefore transposed through a small smem buffer so that 4 (bf16
      // planes) or 4 (fp32, in two 16-column halves) consecutive lanes cover one contiguous 64-byte row segment:
      // every global transaction is a fully written 32-byte sector and an instruction touches 8 rows instead of 32.
      auto store_rows_64B = [&](const uint32_t (&w)[16], uint8_t* base, size_t row_byte_off) {
        uint4* srow = reinterpret_cast<uint4*>(stg + lane * 80);
#pragma unroll
        for (int j = 0; j < 4; ++j) srow[j] = make_uint4(w[4 * j], w[4 * j + 1], w[4 * j + 2], w[4 * j + 3]);
        __syncwarp();
        const uint32_t off_lo = (uint32_t)row_byte_off, off_hi = (uint32_t)(row_byte_off >> 32);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + (lane >> 2), piece = lane & 3;
          const uint4 val = *reinterpret_cast<const uint4*>(stg + rr * 80 + piece * 16);
          const size_t o = ((size_t)__shfl_sync(0xffffffffu, off_hi, rr) << 32) | __shfl_sync(0xffffffffu, off_lo, rr);
          if ((okmask >> rr) & 1u) *reinterpret_cast<uint4*>(base + o + piece * 16) = val;
        }
        __syncwarp();
      };
      auto load_rows_64B = [&](uint32_t (&w)[16], const uint8_t* base, size_t row_byte_off) {
        const uint32_t off_lo = (uint32_t)row_byte_off, off_hi = (uint32_t)(row_byte_off >> 32);
#pragma unroll
        for (int it = 0; it < 4; ++it) {
          const int rr = it * 8 + (lane >> 2), piece = lane & 3;
          const size_t o = ((size_t)__shfl_sync(0xffffffffu, off_hi, rr) << 32) | __shfl_sync(0xffffffffu, off_lo, rr);
          uint4 val = make_uint4(0, 0, 0, 0);
          if ((okmask >> rr) & 1u) val = *reinterpret_cast<const uint4*>(base + o + piece * 16);
          *reinterpret_cast<uint4*>(stg + rr * 80 + piece * 16) = val;
        }
        __syncwarp();
        const uint4* srow = reinterpret_cast<const uint4*>(stg + lane * 80);
#pragma unroll
        for (int j = 0; j < 4; ++j) { const uint4 t = srow[j]; w[4 * j] = t.x; w[4 * j + 1] = t.y; w[4 * j + 2] = t.z; w[4 * j + 3] = t.w; }
        __syncwarp();
      };

      // kSwap: thread = output channel m, the 32 columns of a chunk are 32 consecutive output pixels; every value is
      // transposed through the warp's smem buffer so that a pixel's 32 channels leave as one 64-byte NHWC segment
      auto process_swapped = [&](uint32_t (&v32)[32], int c0) {
        const size_t pix = (size_t)(n0 + c0);
        const size_t cbase = (size_t)(mt * kBM + q * 32);
        const float bias_r = __ldg(p.bias + m);
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) v[j] = __uint_as_float(v32[j]) + bias_r;
        auto rows_in = [&](const uint16_t* plane) {          // v[j] += plane[pix + j][channel of this lane]
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rr = it * 8 + (lane >> 2), piece = lane & 3;
            *reinterpret_cast<uint4*>(stg + rr * 80 + piece * 16) =
                *reinterpret_cast<const uint4*>(reinterpret_cast<const uint8_t*>(plane) + ((pix + rr) * p.M + cbase) * 2 + piece * 16);
          }
          __syncwarp();
#pragma unroll
          for (int j = 0; j < 32; ++j)
            v[j] += __uint_as_float((uint32_t)*reinterpret_cast<const uint16_t*>(stg + j * 80 + lane * 2) << 16);
          __syncwarp();
        };
        if (kMode == GEMM_PLANES_ADD_RELU) { rows_in(p.res_hi); rows_in(p.res_lo); }
        if (kMode == GEMM_PLANES_RELU || kMode == GEMM_PLANES_ADD_RELU) {
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        auto rows_out = [&](uint16_t* plane, bool low) {
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const __nv_bfloat16 h = __float2bfloat16_rn(v[j]);
            const __nv_bfloat16 o = low ? __float2bfloat16_rn(v[j] - __bfloat162float(h)) : h;
            *reinterpret_cast<uint16_t*>(stg + j * 80 + lane * 2) = __bfloat16_as_ushort(o);
          }
          __syncwarp();
#pragma unroll
          for (int it = 0; it < 4; ++it) {
            const int rr = it * 8 + (lane >> 2), piece = lane & 3;
            *reinterpret_cast<uint4*>(reinterpret_cast<uint8_t*>(plane) + ((pix + rr) * p.M + cbase) * 2 + piece * 16) =
                *reinterpret_cast<const uint4*>(stg + rr * 80 + piece * 16);
          }
          __syncwarp();
        };
        rows_out(p.out_hi, false);
        rows_out(p.out_lo, true);
      };

      auto process = [&](uint32_t (&v32)[32], int c0) {
        if constexpr (kSwap) { process_swapped(v32, c0); return; }
        const int n = n0 + c0;
        float v[32];
#pragma unroll
        for (int j = 0; j < 32; ++j)
          v[j] = (p.acc_scale != 0.f ? __uint_as_float(v32[j]) * p.acc_scale : __uint_as_float(v32[j])) + sb[c0 + j];
        if (kMode == GEMM_PLANES || kMode == GEMM_PLANES_GELU || kMode == GEMM_QKV_HEADS || kMode == GEMM_PLANES_RELU ||
            kMode == GEMM_PLANES_ADD_RELU) {
          uint32_t hi[16], lo[16];
          if (kMode == GEMM_PLANES_ADD_RELU) {          // BasicBlock: relu(shortcut + bn2(conv2(.)))   (resnet.py:45-50)
            const size_t rb = (out_row * p.N + n) * 2;
            load_rows_64B(hi, reinterpret_cast<const uint8_t*>(p.res_hi), rb);
            load_rows_64B(lo, reinterpret_cast<const uint8_t*>(p.res_lo), rb);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              v[2 * j] += __uint_as_float(hi[j] << 16) + __uint_as_float(lo[j] << 16);
              v[2 * j + 1] += __uint_as_float(hi[j] & 0xffff0000u) + __uint_as_float(lo[j] & 0xffff0000u);
            }
          }
#pragma unroll
          for (int j = 0; j < 32; j += 2) {
            float a = v[j], b = v[j + 1];
            if (kMode == GEMM_PLANES_GELU) { a = gelu_erf(a); b = gelu_erf(b); }
            if (kMode == GEMM_PLANES_RELU || kMode == GEMM_PLANES_ADD_RELU) { a = fmaxf(a, 0.f); b = fmaxf(b, 0.f); }
            if constexpr (kF16) {                    // saturating: a value beyond the fp16 range stays finite (and wrong) instead of inf
              a = fminf(fmaxf(a, -65504.f), 65504.f);
              b = fminf(fmaxf(b, -65504.f), 65504.f);
              const __half ah = __float2half_rn(a), bh = __float2half_rn(b);
              hi[j >> 1] = (uint32_t)__half_as_ushort(ah) | ((uint32_t)__half_as_ushort(bh) << 16);
              lo[j >> 1] = (uint32_t)__half_as_ushort(__float2half_rn(a - __half2float(ah))) |
                           ((uint32_t)__half_as_ushort(__float2half_rn(b - __half2float(bh))) << 16);
            } else {
              const __nv_bfloat16 ah = __float2bfloat16_rn(a), bh = __float2bfloat16_rn(b);
              hi[j >> 1] = pack_bf16(ah, bh);
              lo[j >> 1] = pack_bf16(__float2bfloat16_rn(a - __bfloat162float(ah)), __float2bfloat16_rn(b - __bfloat162float(bh)));
            }
          }
          size_t dst = out_row * p.N + n;
          if (kMode == GEMM_QKV_HEADS) {   // head-major: [q|k|v][crop][head][token][64] so that attention tiles are contiguous
            const int which = n >> 10, head = (n & 1023) >> 6, d0 = n & 63;
            const int img = m / p.tokens_per_img, tok = m - img * p.tokens_per_img;
            dst = ((((size_t)which * p.qkv_crop_stride + img) * 16 + head) * p.tokens_per_img + tok) * 64 + d0;
          }
          store_rows_64B(hi, reinterpret_cast<uint8_t*>(p.out_hi), dst * 2);
          store_rows_64B(lo, reinterpret_cast<uint8_t*>(p.out_lo), dst * 2);
        } else if (kMode == GEMM_SCALE_RESIDUAL) {      // x += gamma * (acc + bias)   (blocks: ls1 / ls2 + residual)
          const size_t rowb = (out_row * p.N + n) * 4;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            uint32_t w[16];
            load_rows_64B(w, reinterpret_cast<const uint8_t*>(p.x), rowb + half * 64);
#pragma unroll
            for (int j = 0; j < 16; ++j)
              w[j] = __float_as_uint(__uint_as_float(w[j]) + sg[c0 + half * 16 + j] * v[half * 16 + j]);
            store_rows_64B(w, reinterpret_cast<uint8_t*>(p.x), rowb + half * 64);
          }
        } else if (kMode == GEMM_ROWS_F32 || kMode == GEMM_ROWS_F32_RELU) {   // plain fp32 rows (last 1x1 convolution of the IST
          const size_t rowb = (out_row * p.N + n) * 4;                          // trunk; second hidden layer of the IST MLP)
          const float floor_v = kMode == GEMM_ROWS_F32_RELU ? 0.f : -INFINITY;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            uint32_t w[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) w[j] = __float_as_uint(fmaxf(v[half * 16 + j], floor_v));
            store_rows_64B(w, reinterpret_cast<uint8_t*>(p.x), rowb + half * 64);
          }
        } else {                                          // GEMM_PATCH_EMBED
          const size_t rowb = (out_row * p.N + n) * 4;
#pragma unroll
          for (int half = 0; half < 2; ++half) {
            uint32_t w[16];
#pragma unroll
            for (int j = 0; j < 16; ++j)
              w[j] = __float_as_uint(v[half * 16 + j] + (row_ok ? __ldg(pos_row + n + half * 16 + j) : 0.f));
            store_rows_64B(w, reinterpret_cast<uint8_t*>(p.x), rowb + half * 64);
          }
        }
      };

      const float* arow = acc_s + r * kAccPitch + ch * half_cols;
      for (int c0 = 0; c0 < half_cols; c0 += 32) {
        uint32_t v[32];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const uint4 t = *reinterpret_cast<const uint4*>(arow + c0 + 4 * j);
          v[4 * j] = t.x; v[4 * j + 1] = t.y; v[4 * j + 2] = t.z; v[4 * j + 3] = t.w;
        }
        process(v, c0);
      }
      // the ring may take the next tile's operands: order these generic-proxy accesses before the TMA writes
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&tail.ring_free_bar);
      if (e == 0 && lane == 0) GSTAMP(unit * 4 + 3);
    }
  }
}

cudaError_t read_gemm_stamps(long long* host64) { return cudaMemcpyFromSymbol(host64, g_gemm_stamp, sizeof(long long) * 64); }

namespace {
template <bool kSwap, int kTileN, bool kF16, int kMode>
cudaError_t launch_mode(const CUtensorMap& a_hi, const CUtensorMap& a_lo, const CUtensorMap& w_hi, const CUtensorMap& w_lo,
                        const GemmParams& p, int grid, cudaStream_t stream) {
  auto kernel = vit_gemm_kernel<kSwap, kTileN, kF16, kMode>;
  static bool configured = false;                  // one flag per instantiation
  if (!configured) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
    if (e != cudaSuccess) return e;
    configured = true;
  }
  return launch_ex(kernel, dim3(grid), dim3(kThreads), kSmemBytes, stream, 1, true, a_hi, a_lo, w_hi, w_lo, p);
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
