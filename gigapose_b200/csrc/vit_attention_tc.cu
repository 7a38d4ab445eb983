// Multi-head self-attention of the ViT-L/14 forward on TMA + wgmma (row a1; 257 tokens, 16 heads x 64).
//
// One CTA per (crop, head) item.  K and V of the head (272 key rows: 257 + padding) and the first 256 query rows are
// TMA-staged into shared memory as bf16 hi/lo planes (SWIZZLE_128B, 128-byte rows); V lands while S and the softmax
// of the first query tiles run.  Two consumer warpgroups take two 64-row query tiles each:
//   S = Q K^T          wgmma SS, m64 n256 + n16, K=64    (A = Q tile, B = K, both K-major)  -> registers
//   softmax            in registers: a lane quad holds a query row; fp32 max / ex2 / sum, P split into bf16 hi/lo pairs
//                      whose register layout is the A operand layout of the next product
//   O = P V            wgmma RS, m64 n64, K=272           (A = P from registers, B = V as MN-major operand)
//   epilogue           divide by the row sum, store bf16 hi/lo planes (A operand of the proj GEMM)
// Both products use the fp32-faithful split: S = Qh Kh + Qh Kl + Ql Kh, O = Ph Vh + Ph Vl + Pl Vh.
// The 257th query row (token 256) would cost a fifth 64-row tile; one extra warp computes it with fp32 FMAs from the
// same shared-memory K / V planes while the tensor cores run.
// Warp roles: warps 0-7 wgmma + softmax + epilogue, warp 8 TMA producer (one lane) and then token 256.
#include "gigapose_kernels.h"
#include "common.cuh"
#include "wgmma.cuh"
#include <cuda_bf16.h>

namespace gp {

namespace {

constexpr int kTok = 257, kDim = 1024, kHeads = 16, kHd = 64;
constexpr int kKeys = 272;                         // 17 x 16
constexpr int kRow = 128;                          // bytes per smem row (64 bf16) = SWIZZLE_128B span
constexpr int kKVPlane = kKeys * kRow;             // 34 KB
constexpr int kQPlane = 256 * kRow;                // 32 KB: query rows 0..255
constexpr int kQTiles = 4;                         // 64-row tiles: tokens 0..255 on the tensor path; token 256 on one SIMT warp
constexpr int kMmaWarps = 8;
constexpr int kThreads = (kMmaWarps + 1) * 32;

struct __align__(8) AttnTail {
  uint64_t qk_full, v_full;
};
constexpr int kSmem = 1024 + 4 * kKVPlane + 2 * kQPlane + sizeof(AttnTail);

// (a, b) -> packed bf16x2 hi word (a in the low half) and the bf16x2 of the residuals: 6 instructions per pair
__device__ __forceinline__ void split_pair(float a, float b, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(b), "f"(a));
  const float ra = a - __uint_as_float(hi << 16), rb = b - __uint_as_float(hi & 0xffff0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(rb), "f"(ra));
}
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
// exp(x / 8) = 2^(x * log2(e) / 8); the 1/sqrt(64) logit scale is folded into the constant
constexpr float kExpScale = 0.125f * 1.4426950408889634f;
// fp32 value of element `col` of row `row` in a [rows][64] bf16 hi/lo tile stored with the 128-byte TMA swizzle
// (`lo` may be null: plain bf16 mode)
__device__ __forceinline__ float2 ld_pair_sw128(const uint8_t* hi, const uint8_t* lo, int row, int col) {
  const uint32_t off = (uint32_t)row * 128u + ((((uint32_t)col >> 3) ^ ((uint32_t)row & 7u)) << 4) + (((uint32_t)col & 7u) << 1);
  const uint32_t h = *reinterpret_cast<const uint32_t*>(hi + off);
  const uint32_t l = lo ? *reinterpret_cast<const uint32_t*>(lo + off) : 0u;
  return make_float2(__uint_as_float(h << 16) + __uint_as_float(l << 16),
                     __uint_as_float(h & 0xffff0000u) + __uint_as_float(l & 0xffff0000u));
}

}  // namespace

// cycle stamps of CTA 0 (diagnostics: gp_debug_attention_timeline): [0] start, [1] Q / K landed, [2 + wg] warpgroup done
__device__ long long g_attn_stamp[32];
#define STAMP(i) do { if (blockIdx.x == 0) g_attn_stamp[i] = clock64(); } while (0)

template <int kPasses>        // 3 = fp32-faithful split products, 1 = plain bf16 (a template parameter: the other mode's code
__global__ void __launch_bounds__(kThreads, 1)   // and registers stay out of the instruction stream)
attention_tc_kernel(const __grid_constant__ CUtensorMap tm_hi_128, const __grid_constant__ CUtensorMap tm_lo_128,
                    const __grid_constant__ CUtensorMap tm_hi_16, const __grid_constant__ CUtensorMap tm_lo_16,
                    const __nv_bfloat16* __restrict__ qkv_hi, const __nv_bfloat16* __restrict__ qkv_lo,
                    __nv_bfloat16* __restrict__ out_hi, __nv_bfloat16* __restrict__ out_lo, int crop_stride) {
  constexpr int passes = kPasses;
  constexpr int np = passes == 3 ? 2 : 1;
  extern __shared__ uint8_t smem_raw[];
  pdl_trigger();
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint8_t* sK[2] = {smem, smem + kKVPlane};                                   // hi, lo
  uint8_t* sV[2] = {smem + 2 * kKVPlane, smem + 3 * kKVPlane};
  uint8_t* sQ[2] = {smem + 4 * kKVPlane, smem + 4 * kKVPlane + kQPlane};
  AttnTail& tail = *reinterpret_cast<AttnTail*>(smem + 4 * kKVPlane + 2 * kQPlane);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // item -> (crop, head) and the first rows of its operands: head-major planes [q|k|v][crop][head][token][64]
  const int item = blockIdx.x;
  const int img = item / kHeads, head = item % kHeads;
  const int row0 = img * kTok;                       // first token row of this crop in the [M, 1024] output planes
  const int rq = ((0 * crop_stride + img) * kHeads + head) * kTok;
  const int rk = ((1 * crop_stride + img) * kHeads + head) * kTok;
  const int rv = ((2 * crop_stride + img) * kHeads + head) * kTok;

  if (threadIdx.x == 0) {
    mbar_init(&tail.qk_full, 1);
    mbar_init(&tail.v_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();                                        // q / k / v planes come from the QKV GEMM launched before
  if (threadIdx.x == 0) STAMP(0);

  if (warp == kMmaWarps) {
    // ============================== TMA producer (one lane), then token 256 ==============================
    if (lane == 0) {
      tma_prefetch_desc(&tm_hi_128); tma_prefetch_desc(&tm_hi_16);
      if (np == 2) { tma_prefetch_desc(&tm_lo_128); tma_prefetch_desc(&tm_lo_16); }
      mbar_arrive_expect_tx(&tail.qk_full, (uint32_t)(np * (kQPlane + kKVPlane)));
      for (int pl = 0; pl < np; ++pl) {
        const CUtensorMap* m128 = pl ? &tm_lo_128 : &tm_hi_128;
        const CUtensorMap* m16 = pl ? &tm_lo_16 : &tm_hi_16;
        tma_load_2d(sQ[pl], m128, &tail.qk_full, 0, rq);
        tma_load_2d(sQ[pl] + 128 * kRow, m128, &tail.qk_full, 0, rq + 128);
        tma_load_2d(sK[pl], m128, &tail.qk_full, 0, rk);
        tma_load_2d(sK[pl] + 128 * kRow, m128, &tail.qk_full, 0, rk + 128);
        tma_load_2d(sK[pl] + 256 * kRow, m16, &tail.qk_full, 0, rk + 256);
      }
      mbar_arrive_expect_tx(&tail.v_full, (uint32_t)(np * kKVPlane));
      for (int pl = 0; pl < np; ++pl) {
        const CUtensorMap* m128 = pl ? &tm_lo_128 : &tm_hi_128;
        const CUtensorMap* m16 = pl ? &tm_lo_16 : &tm_hi_16;
        tma_load_2d(sV[pl], m128, &tail.v_full, 0, rv);
        tma_load_2d(sV[pl] + 128 * kRow, m128, &tail.v_full, 0, rv + 128);
        tma_load_2d(sV[pl] + 256 * kRow, m16, &tail.v_full, 0, rv + 256);
      }
    }
    __syncwarp();
    // token 256 with fp32 FMAs from the smem planes
    __shared__ float s_p[kKeys];
    __shared__ float s_q[kHd];
    {
    // q (64 values): lane loads q[2*lane], q[2*lane+1] straight from the planes and shares them through smem
    const size_t qoff = (size_t)(rq + 256) * kHd + 2 * lane;
    const uint32_t qh = *reinterpret_cast<const uint32_t*>(qkv_hi + qoff);
    const uint32_t ql = passes == 3 ? *reinterpret_cast<const uint32_t*>(qkv_lo + qoff) : 0u;
    s_q[2 * lane] = __uint_as_float(qh << 16) + __uint_as_float(ql << 16);
    s_q[2 * lane + 1] = __uint_as_float(qh & 0xffff0000u) + __uint_as_float(ql & 0xffff0000u);
    __syncwarp();
    mbar_wait(&tail.qk_full, 0);
    const uint8_t* klo = passes == 3 ? sK[1] : nullptr;   // bf16 mode: the lo planes are not loaded
    const uint8_t* vlo = passes == 3 ? sV[1] : nullptr;
    // logits: lane handles keys lane, lane+32, ...; one 16-byte chunk (8 channels) of a K row per load
    float sj[9];
    float mx = -INFINITY;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int key = lane + 32 * i;
      float acc = 0.f;
      if (key < kTok) {
#pragma unroll
        for (int ch = 0; ch < 8; ++ch) {
          const uint32_t off = (uint32_t)key * 128u + (((uint32_t)ch ^ ((uint32_t)key & 7u)) << 4);
          const uint4 h4 = *reinterpret_cast<const uint4*>(sK[0] + off);
          const uint4 l4 = klo ? *reinterpret_cast<const uint4*>(klo + off) : make_uint4(0, 0, 0, 0);
          const uint32_t hw[4] = {h4.x, h4.y, h4.z, h4.w}, lw[4] = {l4.x, l4.y, l4.z, l4.w};
#pragma unroll
          for (int w = 0; w < 4; ++w) {
            const float k0 = __uint_as_float(hw[w] << 16) + __uint_as_float(lw[w] << 16);
            const float k1 = __uint_as_float(hw[w] & 0xffff0000u) + __uint_as_float(lw[w] & 0xffff0000u);
            acc = fmaf(s_q[ch * 8 + 2 * w], k0, acc);
            acc = fmaf(s_q[ch * 8 + 2 * w + 1], k1, acc);
          }
        }
      }
      sj[i] = key < kTok ? acc : -INFINITY;
      mx = fmaxf(mx, sj[i]);
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int key = lane + 32 * i;
      const float pj = key < kTok ? ex2_approx((sj[i] - mx) * kExpScale) : 0.f;
      sum += pj;
      if (key < kKeys) s_p[key] = pj;
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    __syncwarp();                                      // s_p is complete
    mbar_wait(&tail.v_full, 0);
    // output: lane handles d = 2*lane, 2*lane+1 (4 partial accumulators, loads batched by the unroll)
    float o0[4] = {0.f, 0.f, 0.f, 0.f}, o1[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll 8
    for (int key = 0; key < 256; ++key) {
      const float2 vv = ld_pair_sw128(sV[0], vlo, key, 2 * lane);
      const float pj = s_p[key];
      o0[key & 3] = fmaf(pj, vv.x, o0[key & 3]);
      o1[key & 3] = fmaf(pj, vv.y, o1[key & 3]);
    }
    {
      const float2 vv = ld_pair_sw128(sV[0], vlo, 256, 2 * lane);
      o0[0] = fmaf(s_p[256], vv.x, o0[0]);
      o1[0] = fmaf(s_p[256], vv.y, o1[0]);
    }
    const float o0s = (o0[0] + o0[1]) + (o0[2] + o0[3]), o1s = (o1[0] + o1[1]) + (o1[2] + o1[3]);
    const float inv = 1.0f / sum;
    uint32_t h, l;
    split_pair(o0s * inv, o1s * inv, h, l);
    const size_t oo = (size_t)(row0 + 256) * kDim + head * kHd + 2 * lane;
    *reinterpret_cast<uint32_t*>(out_hi + oo) = h;
    *reinterpret_cast<uint32_t*>(out_lo + oo) = l;
    }
  } else {
    // ============================== wgmma + softmax + epilogue (warps 0-7) ==============================
    const int wg = warp >> 2, wl = warp & 3;
    const uint32_t kh = smem_u32(sK[0]), kl = smem_u32(sK[1]), vh = smem_u32(sV[0]), vl = smem_u32(sV[1]);
    mbar_wait(&tail.qk_full, 0);
    if (threadIdx.x == 0) STAMP(1);
    for (int qt = wg; qt < kQTiles; qt += 2) {
      const uint32_t qh = smem_u32(sQ[0] + qt * 64 * kRow), ql = smem_u32(sQ[1] + qt * 64 * kRow);
      // ---- S = Q K^T: keys [0,256) and [256,272)
      float s[128], st[8];
      acc_fence(s); acc_fence(st);
      wgmma_fence();
#pragma unroll
      for (int pass = 0; pass < passes; ++pass) {
        const uint32_t a = pass == 2 ? ql : qh, b = pass == 1 ? kl : kh;
#pragma unroll
        for (int k16 = 0; k16 < 4; ++k16) {
          const uint32_t acc = (pass | k16) != 0 ? 1u : 0u;
          const uint64_t da = wgmma_desc_kmajor<kRow>(a + k16 * 32);
          wgmma_ss_n256_bf16(s, da, wgmma_desc_kmajor<kRow>(b + k16 * 32), acc);
          wgmma_ss_n16_bf16(st, da, wgmma_desc_kmajor<kRow>(b + 256 * kRow + k16 * 32), acc);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(s); acc_fence(st);
      // ---- softmax.  Fragment: rows r0 = 16 wl + lane / 4 (s[4j], s[4j+1], st[..]) and r0 + 8 (s[4j+2], s[4j+3]);
      // columns 8 j + 2 (lane % 4) + {0, 1}.  Of the 16 tail keys only key 256 (lane % 4 == 0, st[0] / st[2]) is real.
      const bool key256 = (lane & 3) == 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) if (!(key256 && (i & 1) == 0 && i < 4)) st[i] = -INFINITY;
      float mx0 = fmaxf(st[0], st[1]), mx1 = fmaxf(st[2], st[3]);
#pragma unroll
      for (int j = 0; j < 32; ++j) {
        mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
        mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
      }
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, off));
        mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, off));
      }
      float sum0 = 0.f, sum1 = 0.f;
      uint32_t ph[68], pl[68];                         // P as packed bf16 pairs: [chunk of 16 keys][4 A-fragment registers]
#pragma unroll
      for (int j = 0; j < 34; ++j) {                   // 8-column groups: 32 of S, 2 of the tail
        const float x0 = j < 32 ? s[4 * j] : st[4 * (j - 32)], x1 = j < 32 ? s[4 * j + 1] : st[4 * (j - 32) + 1];
        const float x2 = j < 32 ? s[4 * j + 2] : st[4 * (j - 32) + 2], x3 = j < 32 ? s[4 * j + 3] : st[4 * (j - 32) + 3];
        const float p0 = ex2_approx((x0 - mx0) * kExpScale), p1 = ex2_approx((x1 - mx0) * kExpScale);
        const float p2 = ex2_approx((x2 - mx1) * kExpScale), p3 = ex2_approx((x3 - mx1) * kExpScale);
        sum0 += p0 + p1;
        sum1 += p2 + p3;
        // A fragment of chunk c = j / 2: {row r0, k 0-7}, {row r0+8, k 0-7}, {row r0, k 8-15}, {row r0+8, k 8-15}
        const int c = j >> 1, h = (j & 1) * 2;
        split_pair(p0, p1, ph[4 * c + h], pl[4 * c + h]);
        split_pair(p2, p3, ph[4 * c + h + 1], pl[4 * c + h + 1]);
      }
#pragma unroll
      for (int off = 1; off <= 2; off <<= 1) {
        sum0 += __shfl_xor_sync(0xffffffffu, sum0, off);
        sum1 += __shfl_xor_sync(0xffffffffu, sum1, off);
      }
      // ---- O = P V over 17 chunks of 16 keys
      if (qt == wg) mbar_wait(&tail.v_full, 0);
      float o[32];
      acc_fence(o);
      wgmma_fence();
#pragma unroll
      for (int c = 0; c < kKeys / 16; ++c) {
        const uint32_t ah[4] = {ph[4 * c], ph[4 * c + 1], ph[4 * c + 2], ph[4 * c + 3]};
        const uint64_t dvh = wgmma_desc_mnmajor_sw128(vh + c * 16 * kRow);
        wgmma_rs_n64_bf16_tb(o, ah, dvh, c != 0 ? 1u : 0u);
        if (passes == 3) {
          const uint32_t al[4] = {pl[4 * c], pl[4 * c + 1], pl[4 * c + 2], pl[4 * c + 3]};
          wgmma_rs_n64_bf16_tb(o, ah, wgmma_desc_mnmajor_sw128(vl + c * 16 * kRow), 1u);
          wgmma_rs_n64_bf16_tb(o, al, dvh, 1u);
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      acc_fence(o);
      // ---- epilogue: O / sum -> bf16 hi/lo planes
      const float inv0 = 1.0f / sum0, inv1 = 1.0f / sum1;
      const int tok0 = qt * 64 + wl * 16 + (lane >> 2);
      const size_t o0 = (size_t)(row0 + tok0) * kDim + head * kHd + 2 * (lane & 3);
      const size_t o1 = o0 + (size_t)8 * kDim;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        uint32_t h, l;
        split_pair(o[4 * j] * inv0, o[4 * j + 1] * inv0, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + o0 + 8 * j) = h;
        *reinterpret_cast<uint32_t*>(out_lo + o0 + 8 * j) = l;
        split_pair(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1, h, l);
        *reinterpret_cast<uint32_t*>(out_hi + o1 + 8 * j) = h;
        *reinterpret_cast<uint32_t*>(out_lo + o1 + 8 * j) = l;
      }
    }
    if (lane == 0 && wl == 0) STAMP(2 + wg);
  }
}

cudaError_t read_attention_stamps(long long* host32) {
  return cudaMemcpyFromSymbol(host32, g_attn_stamp, sizeof(long long) * 32);
}

cudaError_t launch_attention_tc(const CUtensorMap& hi128, const CUtensorMap& lo128, const CUtensorMap& hi16,
                                const CUtensorMap& lo16, const uint16_t* qkv_hi, const uint16_t* qkv_lo, uint16_t* out_hi,
                                uint16_t* out_lo, int b, int crop_stride, int passes, cudaStream_t s) {
  if (b <= 0) return cudaSuccess;
  const int items = b * kHeads;
  const dim3 grid(items);
  auto qh = reinterpret_cast<const __nv_bfloat16*>(qkv_hi), ql = reinterpret_cast<const __nv_bfloat16*>(qkv_lo);
  auto oh = reinterpret_cast<__nv_bfloat16*>(out_hi), ol = reinterpret_cast<__nv_bfloat16*>(out_lo);
  if (passes == 3)
    return launch_ex(attention_tc_kernel<3>, grid, dim3(kThreads), kSmem, s, 1, true, hi128, lo128, hi16, lo16, qh, ql, oh, ol, crop_stride);
  return launch_ex(attention_tc_kernel<1>, grid, dim3(kThreads), kSmem, s, 1, true, hi128, lo128, hi16, lo16, qh, ql, oh, ol, crop_stride);
}

}  // namespace gp
