// Fused query<->template patch-similarity search for sm_90a (row a4 of SURVEY.md §8; replaces
// LocalSimilarity.test, reference src/models/matching.py:188-316 with helpers :63-113).
//
// One work item = one (query b, template n) pair = one 256(t) x 256(s) x 1024(c) similarity tile.
// A persistent CTA per SM walks the item list:
//   warp 0     : TMA producer  -- streams K-blocks of the query / template descriptor planes into a 4-stage smem ring
//   warps 4-11 : two consumer warpgroups -- wgmma (m64 n256 k16, bf16 -> fp32 registers) on query rows [0,64) and
//                [64,128) of a t-half; the two t-halves of a tile run one after the other while the producer already
//                streams the next half's operands.  Epilogue straight from the accumulator registers: masks + threshold
//                (matching.py:234-236), row max/arg-max (t->s) within a lane quad, column max/arg-max (s->t) through a
//                shared-memory atomic max on (value, -t) keys, cycle-consistency / validity masks (matching.py:80-113,
//                247-271) and the per-template score (matching.py:274-278).  The [B,N,256,256] similarity tensor
//                never reaches HBM; per item only a 1.5 KB record + one float are written.
//
// Precision: descriptors are stored as two bf16 planes (hi = bf16(x), lo = bf16(x - hi)); the tile is accumulated
// as hi*hi + hi*lo + lo*hi in fp32 (3 tensor-core passes, ~2^-17 relative operand error), so the thresholded /
// arg-max'ed results agree with the reference's fp32 einsum up to fp32 accumulation-order noise.  `passes = 1`
// runs hi*hi only (plain bf16 tensor-core similarity, 3x less tensor work, not index-exact).
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"
#include "common.cuh"
#include "wgmma.cuh"
#include <cstdio>

namespace gp {

namespace {

constexpr int kP = 256;                         // patches per crop (16 x 16)
constexpr int kC = 1024;                        // descriptor channels
constexpr int kBlockK = 32;                     // bf16 elements per stage row: 64 B = SWIZZLE_64B span
constexpr int kRowBytes = kBlockK * 2;
constexpr int kStages = 4;
constexpr int kHalfRows = 128;                  // t-rows per half tile (two warpgroups of 64)
constexpr int kQPlaneBytes = kHalfRows * kRowBytes;   // 8 KB : 128 query rows x 64 B
constexpr int kTPlaneBytes = kP * kRowBytes;          // 16 KB: 256 template rows x 64 B
constexpr int kStageBytes = 2 * kQPlaneBytes + 2 * kTPlaneBytes;   // q_hi, q_lo, t_hi, t_lo = 48 KB
constexpr int kNumKBlocks = kC / kBlockK;       // 32
constexpr int kEpiWarps = 8;
constexpr int kEpiThreads = kEpiWarps * 32;     // 256
constexpr int kThreads = 4 * 32 + kEpiThreads;  // 384

// Item order: queries (sorted by object) are taken in chunks of kQueryChunk; inside a chunk the template index is the
// outer loop.  CTAs that run together then share template tiles (queries of one object are adjacent) AND touch at
// most kQueryChunk query tiles, so both operands stay L2-resident whatever the batch size (at B = 256 with one query
// per object the plain template-major order re-read every query tile from HBM once per template).
constexpr int kQueryChunk = 32;
__device__ __forceinline__ void decode_item(int item, int B, int T, int& j, int& n) {
  const int per_chunk = kQueryChunk * T;
  const int c = item / per_chunk, r = item - c * per_chunk;
  const int q0 = c * kQueryChunk;
  const int qc = min(kQueryChunk, B - q0);
  n = r / qc;
  j = q0 + (r - n * qc);
}

struct __align__(8) SimSmemTail {
  unsigned long long colkey[kP];                // per column s: max over t of (ord(v) << 32 | 255 - t)
  float smask[kP];                              // template mask sampled at 16x16 (float: alpha masks are not binary)
  float tmask[kP];                              // query mask sampled at 16x16
  float cmax[kP];                               // score_src2tar
  float rmax_s[kP];                             // score_tar2src
  float red[2][kEpiWarps];
  uint8_t cidx[kP];                             // idx_src2tar
  uint8_t ridx_s[kP];                           // idx_tar2src
  uint64_t full_bar[kStages];
  uint64_t empty_bar[kStages];
};

constexpr int kSmemBytes = 1024 /*alignment slack*/ + kStages * kStageBytes + sizeof(SimSmemTail);

}  // namespace

// Work unit of the producer: (item, t-half) = a 128(t) x 256(s) x 1024(c) half tile; the template planes are streamed
// once per half.
// kSigned: sim_threshold <= 0 lets negative values (and -0.0 from masked patches) through the threshold.  The column
// arg-max key then maps the float to an order-preserving uint32 (-0.0 folded into +0.0) instead of taking its bits as
// they are, which orders only values >= +0.0; the row maximum starts at -inf instead of -1.
template <bool kDebug, bool kSigned>
__global__ void __launch_bounds__(kThreads, 1)
sim_search_kernel(const __grid_constant__ CUtensorMap tm_q_hi, const __grid_constant__ CUtensorMap tm_q_lo,
                  const __grid_constant__ CUtensorMap tm_t_hi, const __grid_constant__ CUtensorMap tm_t_lo,
                  SimSearchParams p) {
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_64B atoms repeat every 512 B; keep every plane 1024 B aligned
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  SimSmemTail& tail = *reinterpret_cast<SimSmemTail*>(smem + kStages * kStageBytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int passes = p.passes;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&tail.full_bar[s], 1);
      mbar_init(&tail.empty_bar[s], kEpiWarps);
    }
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    tma_prefetch_desc(&tm_q_hi);
    tma_prefetch_desc(&tm_t_hi);
    if (passes == 3) {
      tma_prefetch_desc(&tm_q_lo);
      tma_prefetch_desc(&tm_t_lo);
    }
  }
  __syncthreads();

  if (warp == 0) {
    // ======================================= TMA producer =======================================
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const uint32_t tx_bytes = (passes == 3 ? 2 : 1) * (kQPlaneBytes + kTPlaneBytes);
      for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
        int j, n;
        decode_item(item, p.B, p.T, j, n);
        const int b = p.perm[j];
        const int t_img = p.q_obj[b] * p.T + n;
        for (int half = 0; half < 2; ++half) {
          for (int kbi = 0; kbi < kNumKBlocks; ++kbi) {
            // the second t-half walks K backwards: the template slabs it needs first are the ones the first half
            // touched last, i.e. the ones most likely still in L2 when nothing else shares the template (B_o = 1)
            const int kb = half == 0 ? kbi : kNumKBlocks - 1 - kbi;
            mbar_wait(&tail.empty_bar[stage], phase ^ 1);
            uint8_t* st = smem + stage * kStageBytes;
            mbar_arrive_expect_tx(&tail.full_bar[stage], tx_bytes);
            // k-block-tiled planes: slab (image, kb) = 256 contiguous 64-byte rows
            const int q_row = (b * kNumKBlocks + kb) * kP + half * kHalfRows;
            const int t_row = (t_img * kNumKBlocks + kb) * kP;
            tma_load_2d(st, &tm_q_hi, &tail.full_bar[stage], 0, q_row);
            tma_load_2d(st + 2 * kQPlaneBytes, &tm_t_hi, &tail.full_bar[stage], 0, t_row);
            if (passes == 3) {
              tma_load_2d(st + 2 * kQPlaneBytes + kTPlaneBytes, &tm_t_lo, &tail.full_bar[stage], 0, t_row);
              tma_load_2d(st + kQPlaneBytes, &tm_q_lo, &tail.full_bar[stage], 0, q_row);
            }
            if (++stage == kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else if (warp >= 4) {
    // ================================ wgmma consumers + epilogue =================================
    const int e = warp - 4;
    const int wg = e >> 2, wl = e & 3;       // warpgroup wg: rows [64 wg, 64 wg + 64) of each half tile
    const int tid = e * 32 + lane;           // 0..255: also "patch owned by this thread" in the per-tile tail
    const float thr = p.sim_threshold;
    int stage = 0;
    uint32_t phase = 0;
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
      int j, n;
      decode_item(item, p.B, p.T, j, n);
      const int b = p.perm[j];
      const size_t rec = (size_t)b * p.T + n;
      tail.smask[tid] = p.bank_mask[((size_t)p.q_obj[b] * p.T + n) * kP + tid];
      tail.tmask[tid] = p.q_mask[(size_t)b * kP + tid];
      tail.colkey[tid] = 0ull;
      named_barrier_sync(1, kEpiThreads);

      for (int half = 0; half < 2; ++half) {
        float acc[kP / 2];
        int prev_stage = -1;
        for (int kb = 0; kb < kNumKBlocks; ++kb) {
          mbar_wait(&tail.full_bar[stage], phase);
          const uint32_t st = smem_u32(smem + stage * kStageBytes);
          const uint32_t q_hi = st + wg * (kQPlaneBytes / 2), q_lo = q_hi + kQPlaneBytes;
          const uint32_t t_hi = st + 2 * kQPlaneBytes, t_lo = t_hi + kTPlaneBytes;
          acc_fence(acc);
          wgmma_fence();
#pragma unroll
          for (int pass = 0; pass < 3; ++pass) {
            if (pass < passes) {
              const uint32_t a = (pass == 2 ? q_lo : q_hi);
              const uint32_t bsm = (pass == 1 ? t_lo : t_hi);
#pragma unroll
              for (int k16 = 0; k16 < kBlockK / 16; ++k16) {
                const uint32_t accum = (kb | pass | k16) != 0 ? 1u : 0u;
                wgmma_ss_n256_bf16(acc, wgmma_desc_kmajor<kRowBytes>(a + k16 * 32), wgmma_desc_kmajor<kRowBytes>(bsm + k16 * 32),
                                   accum);
              }
            }
          }
          wgmma_commit();
          wgmma_wait<1>();                                          // previous k-block retired: its stage is free
          if (prev_stage >= 0 && lane == 0) mbar_arrive(&tail.empty_bar[prev_stage]);
          prev_stage = stage;
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
        acc_fence(acc);
        if (lane == 0) mbar_arrive(&tail.empty_bar[prev_stage]);

        // accumulator fragment: rows t0 = .. + lane/4 and t0 + 8, columns s = 8 j8 + 2 (lane % 4) + {0, 1}
        const int t0 = half * kHalfRows + wg * 64 + wl * 16 + (lane >> 2), t1 = t0 + 8;
        const float tm0 = tail.tmask[t0], tm1 = tail.tmask[t1];
        // thr > 0: all candidates are >= 0 after thresholding -> first max wins
        float rbest0 = kSigned ? -INFINITY : -1.0f, rbest1 = kSigned ? -INFINITY : -1.0f;
        int ridx0 = 0, ridx1 = 0;
#pragma unroll
        for (int j8 = 0; j8 < kP / 8; ++j8) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int s = 8 * j8 + 2 * (lane & 3) + c;
            const float raw0 = acc[4 * j8 + c], raw1 = acc[4 * j8 + 2 + c];
            if (kDebug) {
              const size_t tile = (size_t)n * p.B + j;
              p.debug_tile[(tile * kP + t0) * kP + s] = raw0;
              p.debug_tile[(tile * kP + t1) * kP + s] = raw1;
            }
            const float sm = tail.smask[s];
            float v0 = raw0 * sm, v1 = raw1 * sm;                             // matching.py:234
            v0 = v0 * tm0; v1 = v1 * tm1;                                     // matching.py:235
            v0 = (v0 < thr) ? 0.0f : v0; v1 = (v1 < thr) ? 0.0f : v1;         // matching.py:236
            if (v0 > rbest0) { rbest0 = v0; ridx0 = s; }                      // torch.max(dim=3): first maximum
            if (v1 > rbest1) { rbest1 = v1; ridx1 = s; }
            // torch.max(dim=2): first maximum over t.  v >= 0: float order == uint order; ties -> the smaller t
            const bool second = v1 > v0;
            uint32_t bits = __float_as_uint(second ? v1 : v0);
            if constexpr (kSigned) {
              bits = bits == 0x80000000u ? 0u : bits;                         // -0.0 == +0.0 for torch.max
              bits ^= (uint32_t)((int)bits >> 31) | 0x80000000u;              // order-preserving float -> uint32
            }
            const unsigned long long key = ((unsigned long long)bits << 32) | (unsigned)(255 - (second ? t1 : t0));
            atomicMax(&tail.colkey[s], key);
          }
        }
        // the four lanes of a quad hold the 256 columns of rows t0 / t1 (ties: lower s wins)
#pragma unroll
        for (int off = 1; off <= 2; off <<= 1) {
          const float o0 = __shfl_xor_sync(0xffffffffu, rbest0, off), o1 = __shfl_xor_sync(0xffffffffu, rbest1, off);
          const int i0 = __shfl_xor_sync(0xffffffffu, ridx0, off), i1 = __shfl_xor_sync(0xffffffffu, ridx1, off);
          if (o0 > rbest0 || (o0 == rbest0 && i0 < ridx0)) { rbest0 = o0; ridx0 = i0; }
          if (o1 > rbest1 || (o1 == rbest1 && i1 < ridx1)) { rbest1 = o1; ridx1 = i1; }
        }
        if ((lane & 3) == 0) {
          tail.rmax_s[t0] = rbest0; tail.ridx_s[t0] = (uint8_t)ridx0;
          tail.rmax_s[t1] = rbest1; tail.ridx_s[t1] = (uint8_t)ridx1;
        }
      }
      named_barrier_sync(1, kEpiThreads);
      {
        const unsigned long long key = tail.colkey[tid];
        uint32_t bits = (uint32_t)(key >> 32);
        if constexpr (kSigned) bits = (bits & 0x80000000u) ? (bits ^ 0x80000000u) : ~bits;
        tail.cmax[tid] = __uint_as_float(bits);
        tail.cidx[tid] = (uint8_t)(255u - (uint32_t)(key & 0xffu));
      }
      named_barrier_sync(1, kEpiThreads);

      // matching.py:247-271 for query patch t = tid
      const int t = tid;
      const float rmax = tail.rmax_s[t];
      const int ridx = tail.ridx_s[t];
      const float tm = tail.tmask[t];
      const bool mask_sim = rmax >= thr;
      const int back = tail.cidx[ridx];                                   // idx_src2tar[idx_tar2src[t]]
      const float dx = (float)(back & 15) - (float)(t & 15);
      const float dy = (float)(back >> 4) - (float)(t >> 4);
      const bool mask_cycle = (sqrtf(dx * dx + dy * dy) <= p.patch_threshold) && (tail.cmax[ridx] >= thr);
      // reference quirk kept on purpose: `idx_src2tar != 0` is indexed by s but multiplied position-wise with t
      float mnz = tm * tail.smask[ridx];
      mnz = mnz * (tail.cidx[t] != 0 ? 1.0f : 0.0f);
      mnz = mnz * (ridx != 0 ? 1.0f : 0.0f);
      const float mall = (mask_sim && mask_cycle) ? mnz : 0.0f;
      float s_contrib = rmax * mall, s_mall = mall;
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) {
        s_contrib += __shfl_xor_sync(0xffffffffu, s_contrib, off);
        s_mall += __shfl_xor_sync(0xffffffffu, s_mall, off);
      }
      if (lane == 0) { tail.red[0][e] = s_contrib; tail.red[1][e] = s_mall; }
      p.rec_score[rec * kP + t] = rmax;
      p.rec_idx[rec * kP + t] = (uint8_t)ridx;
      p.rec_valid[rec * kP + t] = (mall != 0.0f) ? 1 : 0;
      named_barrier_sync(1, kEpiThreads);
      if (t == 0) {
        float a = 0.f, m = 0.f;
#pragma unroll
        for (int g = 0; g < kEpiWarps; ++g) { a += tail.red[0][g]; m += tail.red[1][g]; }
        p.sim_avg[rec] = (m > 0.f) ? a / (float)kP : 0.0f;              // matching.py:274-278
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------------------
// top-k template selection (matching.py:279) + compact candidate records
// ------------------------------------------------------------------------------------------------------------
// One CTA per query.  k rounds of block-wide arg-max over the per-template scores; ties break towards the lowest
// template index (torch.topk leaves tie order unspecified).  Emits one compact record per winner:
//   cand_score[b,k] f32, cand_id[b,k] i32 (GLOBAL template id = local * id_stride + id_offset),
//   cand_pts_score[b,k,256] f32, cand_idx[b,k,256] u8, cand_valid[b,k,256] u8
__global__ void __launch_bounds__(256)
topk_select_kernel(TopkSelectParams p) {
  extern __shared__ float s_val[];                 // [T]
  __shared__ float s_wv[8];
  __shared__ int s_wi[8];
  __shared__ int s_win;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int i = tid; i < p.T; i += 256) s_val[i] = p.sim_avg[(size_t)b * p.T + i];
  __syncthreads();
  for (int kk = 0; kk < p.k; ++kk) {
    float bv = -INFINITY;
    int bi = 0x7fffffff;
    for (int i = tid; i < p.T; i += 256) {
      const float v = s_val[i];
      if (v != -INFINITY && (v > bv || (v == bv && i < bi))) { bv = v; bi = i; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { s_wv[warp] = bv; s_wi[warp] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < 8; ++w)
        if (s_wv[w] > bv || (s_wv[w] == bv && s_wi[w] < bi)) { bv = s_wv[w]; bi = s_wi[w]; }
      s_win = bi;
      const size_t o = (size_t)b * p.k + kk;
      if (bi < p.T) {
        p.cand_score[o] = bv;
        p.cand_id[o] = bi * p.id_stride + p.id_offset;
        s_val[bi] = -INFINITY;                     // exclude from later rounds (no score is -inf: they are finite)
      } else {                                     // fewer than k local templates: padding candidate
        p.cand_score[o] = -INFINITY;
        p.cand_id[o] = 0x7fffffff;
      }
    }
    __syncthreads();
    const int win = s_win;
    const size_t o = ((size_t)b * p.k + kk) * kP + tid;
    if (win < p.T) {
      const size_t r = ((size_t)b * p.T + win) * kP + tid;
      p.cand_pts_score[o] = p.rec_score[r];
      p.cand_idx[o] = p.rec_idx[r];
      p.cand_valid[o] = p.rec_valid[r];
    } else {
      p.cand_pts_score[o] = 0.f;
      p.cand_idx[o] = 0;
      p.cand_valid[o] = 0;
    }
    __syncthreads();
  }
}

// Merge G per-shard candidate lists (G = 1 on a single GPU) into the global top-k and expand the winners into the
// reference's output format (matching.py:282-316, format_prediction :29-61):
//   id_src[B,k] i64, score_src[B,k] f32, score_pts[B,k,256] f32, tar_pts/src_pts[B,k,256,2] i64 (-1 = invalid).
// Candidates are laid out [G][B][k]; ordering = score descending, then global template id ascending.
template <typename T>
__device__ __forceinline__ const T* rank_ptr(const T* base, int g, size_t rank_stride_bytes, size_t dense_elems) {
  return rank_stride_bytes ? reinterpret_cast<const T*>(reinterpret_cast<const char*>(base) + (size_t)g * rank_stride_bytes)
                           : base + (size_t)g * dense_elems;
}

__global__ void __launch_bounds__(256)
topk_merge_expand_kernel(TopkMergeParams p) {
  __shared__ int s_sel[32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const int ncand = p.G * p.k;
  const size_t bk = (size_t)p.B * p.k;
  if (tid == 0) {
    // tiny selection sort over <= 64 candidates: score descending, then global template id ascending
    unsigned long long used = 0;
    for (int kk = 0; kk < p.k; ++kk) {
      float bv = 0.f; int bid = 0; int bc = -1;
      for (int c = 0; c < ncand; ++c) {
        if (used >> c & 1ull) continue;
        const int g = c / p.k, j = c - g * p.k;
        const size_t o = (size_t)b * p.k + j;
        const float v = rank_ptr(p.cand_score, g, p.rank_stride_bytes, bk)[o];
        const int id = rank_ptr(p.cand_id, g, p.rank_stride_bytes, bk)[o];
        if (bc < 0 || v > bv || (v == bv && id < bid)) { bv = v; bid = id; bc = c; }
      }
      used |= 1ull << bc;
      s_sel[kk] = bc;
    }
  }
  __syncthreads();
  for (int kk = 0; kk < p.k; ++kk) {
    const int c = s_sel[kk];
    const int g = c / p.k, j = c - g * p.k;
    const size_t o = (size_t)b * p.k + j;
    const size_t dst = (size_t)b * p.k + kk;
    if (tid == 0) {
      p.id_src[dst] = (long long)rank_ptr(p.cand_id, g, p.rank_stride_bytes, bk)[o];
      p.score_src[dst] = rank_ptr(p.cand_score, g, p.rank_stride_bytes, bk)[o];
    }
    const int t = tid;
    const bool valid = rank_ptr(p.cand_valid, g, p.rank_stride_bytes, bk * kP)[o * kP + t] != 0;
    const int s = rank_ptr(p.cand_idx, g, p.rank_stride_bytes, bk * kP)[o * kP + t];
    p.score_pts[dst * kP + t] = rank_ptr(p.cand_pts_score, g, p.rank_stride_bytes, bk * kP)[o * kP + t];
    longlong2 tp, sp;
    tp.x = valid ? (long long)(t & 15) : -1ll;
    tp.y = valid ? (long long)(t >> 4) : -1ll;
    sp.x = valid ? (long long)(s & 15) : -1ll;
    sp.y = valid ? (long long)(s >> 4) : -1ll;
    reinterpret_cast<longlong2*>(p.tar_pts)[dst * kP + t] = tp;
    reinterpret_cast<longlong2*>(p.src_pts)[dst * kP + t] = sp;
    if (p.out_rel_scale && p.cand_rel_scale)
      p.out_rel_scale[dst * kP + t] = rank_ptr(p.cand_rel_scale, g, p.rank_stride_bytes, bk * kP)[o * kP + t];
    if (p.out_rel_inplane && p.cand_rel_inplane)
      reinterpret_cast<float2*>(p.out_rel_inplane)[dst * kP + t] =
          reinterpret_cast<const float2*>(rank_ptr(p.cand_rel_inplane, g, p.rank_stride_bytes, bk * kP * 2))[o * kP + t];
  }
}

// ------------------------------------------------------------------------------------------------------------
// host-side launchers
// ------------------------------------------------------------------------------------------------------------
cudaError_t launch_sim_search(const CUtensorMap& q_hi, const CUtensorMap& q_lo, const CUtensorMap& t_hi,
                              const CUtensorMap& t_lo, const SimSearchParams& p, int num_sms, cudaStream_t stream) {
  if (p.num_items <= 0) return cudaSuccess;
  const int grid = p.num_items < num_sms ? p.num_items : num_sms;
  const bool sign = !(p.sim_threshold > 0.f);         // negative values survive the threshold
  auto kernel = p.debug_tile ? (sign ? sim_search_kernel<true, true> : sim_search_kernel<true, false>)
                             : (sign ? sim_search_kernel<false, true> : sim_search_kernel<false, false>);
  return launch_ex(kernel, grid, kThreads, kSmemBytes, stream, 1, false, q_hi, q_lo, t_hi, t_lo, p);
}

cudaError_t launch_topk_select(const TopkSelectParams& p, cudaStream_t stream) {
  if (p.B <= 0) return cudaSuccess;
  if (p.T > GP_MAX_NUM_TEMPLATES) return cudaErrorInvalidValue;     // s_val[T] must fit the default 48 KiB
  return launch_ex(topk_select_kernel, p.B, 256, p.T * sizeof(float), stream, 1, false, p);
}

cudaError_t launch_topk_merge_expand(const TopkMergeParams& p, cudaStream_t stream) {
  if (p.B <= 0) return cudaSuccess;
  return launch_ex(topk_merge_expand_kernel, p.B, 256, 0, stream, 1, false, p);
}

int sim_search_smem_bytes() { return kSmemBytes; }

}  // namespace gp
