// Per-correspondence scale / in-plane regression (row a5 of SURVEY.md §8; replaces ISTNet.inference
// ist_net.py:97-120, gather utils/batch.py:46-73 and the two Regressor MLP heads ist_net.py:140-155).
//
// For every valid correspondence (b, k, t) a 512-vector cat(query IST descriptor at tar_pt, template IST descriptor at
// src_pt) goes through   scale: 512 -> 512 -> 256 -> 1      in-plane: 512 -> 512 -> 256 -> 2 (tanh).
// The data-dependent row set (boolean-mask indexing + host syncs in the reference) becomes a device-side compaction
// (no host round trip: grids are sized for the worst case and idle tiles exit on the device-side row count).
// fp32 SIMT GEMMs with the gather fused into the A-tile loader: the downstream RANSAC inlier test (<= 14 px) is a
// knife edge on these outputs, so this stage stays in fp32 rather than on bf16 tensor cores.
#include "gigapose_kernels.h"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace gp {

namespace {

constexpr int kP = 256;
constexpr int kIstC = 256;
constexpr int BM = 64, BN = 64, BK = 16;

__global__ void __launch_bounds__(256)
mlp_compact_kernel(IstMlpParams p, int total) {
  const int i = blockIdx.x * 256 + threadIdx.x;
  if (i >= total) return;
  const long long sx = p.src_pts[2 * (size_t)i], sy = p.src_pts[2 * (size_t)i + 1];
  const bool valid = (sx != -1) && (sy != -1);
  p.rel_scale[i] = -1000.0f;                              // ist_net.py:110-113
  p.rel_inplane[2 * (size_t)i] = -1000.0f;
  p.rel_inplane[2 * (size_t)i + 1] = -1000.0f;
  // warp-aggregated append
  const unsigned bal = __ballot_sync(0xffffffffu, valid);
  const int lane = threadIdx.x & 31;
  int base = 0;
  if (lane == 0 && bal) base = atomicAdd(p.row_count, __popc(bal));
  base = __shfl_sync(0xffffffffu, base, 0);
  if (valid) p.row_ids[base + __popc(bal & ((1u << lane) - 1))] = i;
}

// C[r, n] = relu(A[r,:] . W[n,:] + bias[n]),  A rows either gathered (layer 1) or dense (layer 2)
template <bool kGather>
__global__ void __launch_bounds__(256)
mlp_gemm_kernel(IstMlpParams p, const float* __restrict__ Wa, const float* __restrict__ ba,
                const float* __restrict__ Wb, const float* __restrict__ bb,   // second head (layer 1: cols >= 512)
                const float* __restrict__ Adense, int lda, int K, float* __restrict__ out, int ldo) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Ws[BK][BN + 4];
  __shared__ long long s_off0[BM], s_off1[BM];
  const int M = *p.row_count;
  const int r0 = blockIdx.x * BM;
  if (r0 >= M) return;
  const int tid = threadIdx.x;
  // blockIdx.z = head for the dense (layer 2) variant
  const int head = kGather ? 0 : blockIdx.z;
  int n0 = blockIdx.y * BN;
  const float* W;
  const float* bias;
  int out_col0;
  if (kGather) {                         // N = 1024 = [scale head 512 | inplane head 512]
    const bool second = n0 >= 512;
    W = second ? Wb : Wa;
    bias = second ? bb : ba;
    out_col0 = n0;
    n0 = second ? n0 - 512 : n0;
  } else {                               // per head: A = hidden1[:, head*512 : +512], N = 256
    W = head ? Wb : Wa;
    bias = head ? bb : ba;
    out_col0 = head * 256 + n0;
  }
  if (kGather) {
    if (tid < BM) {
      const int r = r0 + tid;
      long long o0 = 0, o1 = 0;
      if (r < M) {
        const int flat = p.row_ids[r];
        const int t = flat & (kP - 1);
        const int bk = flat >> 8;
        const int b = bk / p.k;
        const long long tx = p.tar_pts[2 * (size_t)flat], ty = p.tar_pts[2 * (size_t)flat + 1];
        const long long sx = p.src_pts[2 * (size_t)flat], sy = p.src_pts[2 * (size_t)flat + 1];
        const long long lid = (p.id_src[bk] - p.id_offset) / p.id_stride;
        (void)t;
        o0 = ((long long)b * kP + (ty * 16 + tx)) * kIstC;
        o1 = (((long long)p.q_obj[b] * p.T + lid) * kP + (sy * 16 + sx)) * kIstC;
      }
      s_off0[tid] = o0;
      s_off1[tid] = o1;
    }
    __syncthreads();
  }
  const int lrow = tid >> 2, lk = (tid & 3) * 4;
  const int ty = tid >> 4, tx = tid & 15;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < K; k0 += BK) {
    float4 a4;
    if (kGather) {
      const int kk = k0 + lk;                                    // a BK chunk never straddles the 256 boundary
      const float* src = (kk < kIstC) ? (p.q_ist + s_off0[lrow] + kk) : (p.bank_ist + s_off1[lrow] + (kk - kIstC));
      a4 = (r0 + lrow < M) ? *reinterpret_cast<const float4*>(src) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      a4 = (r0 + lrow < M) ? *reinterpret_cast<const float4*>(Adense + (size_t)(r0 + lrow) * lda + head * 512 + k0 + lk)
                           : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    const float4 w4 = *reinterpret_cast<const float4*>(W + (size_t)(n0 + lrow) * K + k0 + lk);
    As[lk + 0][lrow] = a4.x; As[lk + 1][lrow] = a4.y; As[lk + 2][lrow] = a4.z; As[lk + 3][lrow] = a4.w;
    Ws[lk + 0][lrow] = w4.x; Ws[lk + 1][lrow] = w4.y; Ws[lk + 2][lrow] = w4.z; Ws[lk + 3][lrow] = w4.w;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&Ws[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w}, wv[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], wv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty * 4 + i;
    if (r < M) {
      float4 o;
      o.x = fmaxf(acc[i][0] + bias[n0 + tx * 4 + 0], 0.f);
      o.y = fmaxf(acc[i][1] + bias[n0 + tx * 4 + 1], 0.f);
      o.z = fmaxf(acc[i][2] + bias[n0 + tx * 4 + 2], 0.f);
      o.w = fmaxf(acc[i][3] + bias[n0 + tx * 4 + 3], 0.f);
      *reinterpret_cast<float4*>(out + (size_t)r * ldo + out_col0 + tx * 4) = o;
    }
  }
}

// last layers: scale = h2[0:256].w + b ; (cos,sin) = tanh(h2[256:512].W[2,256] + b) ; one warp per row, scatter
__global__ void __launch_bounds__(256)
mlp_head_kernel(IstMlpParams p, IstMlpWeights w, int max_rows) {
  const int M = *p.row_count;
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= M || r >= max_rows) return;
  const float* h = p.hidden2 + (size_t)r * 512;
  float s = 0.f, c0 = 0.f, c1 = 0.f;
  for (int i = lane; i < 256; i += 32) {
    s = fmaf(h[i], w.s_w3[i], s);
    const float v = h[256 + i];
    c0 = fmaf(v, w.i_w3[i], c0);
    c1 = fmaf(v, w.i_w3[256 + i], c1);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    c0 += __shfl_xor_sync(0xffffffffu, c0, off);
    c1 += __shfl_xor_sync(0xffffffffu, c1, off);
  }
  if (lane == 0) {
    const int flat = p.row_ids[r];
    s += w.s_b3[0];
    c0 += w.i_b3[0];
    c1 += w.i_b3[1];
    if (w.use_tanh) { c0 = tanhf(c0); c1 = tanhf(c1); }
    p.rel_scale[flat] = s;
    p.rel_inplane[2 * (size_t)flat] = c0;
    p.rel_inplane[2 * (size_t)flat + 1] = c1;
  }
}

// ---- tensor-core form: gather the compacted rows into fp16 hi/lo planes (one warp per valid correspondence) ---------------
__global__ void __launch_bounds__(256)
mlp_gather_planes_kernel(IstMlpParams p, __half* __restrict__ a_hi, __half* __restrict__ a_lo, int max_rows) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= *p.row_count || r >= max_rows) return;
  const int flat = p.row_ids[r];                              // (b, k, t) of this valid correspondence
  const int bk = flat >> 8, b = bk / p.k;
  const long long tx = p.tar_pts[2 * (size_t)flat], ty = p.tar_pts[2 * (size_t)flat + 1];
  const long long sx = p.src_pts[2 * (size_t)flat], sy = p.src_pts[2 * (size_t)flat + 1];
  const long long lid = (p.id_src[bk] - p.id_offset) / p.id_stride;
  const float* q = p.q_ist + ((long long)b * kP + (ty * 16 + tx)) * kIstC;
  const float* t = p.bank_ist + (((long long)p.q_obj[b] * p.T + lid) * kP + (sy * 16 + sx)) * kIstC;
#pragma unroll
  for (int part = 0; part < 2; ++part) {                  // columns [0,256) = query descriptor, [256,512) = template descriptor
    const float* src = part ? t : q;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int c = (lane + 32 * i) * 4;
      const float4 v = *reinterpret_cast<const float4*>(src + c);
      const float x[4] = {v.x, v.y, v.z, v.w};
      // IEEE fp16 hi / lo: 22 significant bits for these O(1) descriptors (bf16 pairs carry 16), same tensor rate
      __half h[4], l[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float xs = fminf(fmaxf(x[j], -65504.f), 65504.f);            // saturate instead of inf
        h[j] = __float2half_rn(xs);
        l[j] = __float2half_rn(xs - __half2float(h[j]));
      }
      const size_t o = (size_t)r * 512 + part * 256 + c;
      *reinterpret_cast<uint2*>(a_hi + o) = make_uint2((uint32_t)__half_as_ushort(h[0]) | ((uint32_t)__half_as_ushort(h[1]) << 16),
                                                       (uint32_t)__half_as_ushort(h[2]) | ((uint32_t)__half_as_ushort(h[3]) << 16));
      *reinterpret_cast<uint2*>(a_lo + o) = make_uint2((uint32_t)__half_as_ushort(l[0]) | ((uint32_t)__half_as_ushort(l[1]) << 16),
                                                       (uint32_t)__half_as_ushort(l[2]) | ((uint32_t)__half_as_ushort(l[3]) << 16));
    }
  }
}

// last layers on the compacted rows: one warp per row, fp32, scattered back to (b,k,t)
__global__ void __launch_bounds__(256)
mlp_head_rows_kernel(IstMlpParams p, IstMlpWeights w, const float* __restrict__ h2s, const float* __restrict__ h2i, int max_rows) {
  const int r = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= *p.row_count || r >= max_rows) return;
  const float* hs = h2s + (size_t)r * 256;
  const float* hi = h2i + (size_t)r * 256;
  float s = 0.f, c0 = 0.f, c1 = 0.f;
  for (int i = lane; i < 256; i += 32) {
    s = fmaf(hs[i], w.s_w3[i], s);
    const float v = hi[i];
    c0 = fmaf(v, w.i_w3[i], c0);
    c1 = fmaf(v, w.i_w3[256 + i], c1);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, off);
    c0 += __shfl_xor_sync(0xffffffffu, c0, off);
    c1 += __shfl_xor_sync(0xffffffffu, c1, off);
  }
  if (lane == 0) {
    const int flat = p.row_ids[r];
    s += w.s_b3[0];
    c0 += w.i_b3[0];
    c1 += w.i_b3[1];
    if (w.use_tanh) { c0 = tanhf(c0); c1 = tanhf(c1); }
    p.rel_scale[flat] = s;
    p.rel_inplane[2 * (size_t)flat] = c0;
    p.rel_inplane[2 * (size_t)flat + 1] = c1;
  }
}

}  // namespace

cudaError_t launch_mlp_gather_planes(const IstMlpParams& p, uint16_t* a_hi, uint16_t* a_lo, cudaStream_t stream) {
  const int total = p.B * p.k * kP;
  if (total <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(p.row_count, 0, sizeof(int), stream);
  if (e != cudaSuccess) return e;
  // row_ids, row_count, -1000 fill
  if ((e = launch_ex(mlp_compact_kernel, (total + 255) / 256, 256, 0, stream, 1, false, p, total)) != cudaSuccess) return e;
  return launch_ex(mlp_gather_planes_kernel, (total + 7) / 8, 256, 0, stream, 1, false, p, reinterpret_cast<__half*>(a_hi),
                   reinterpret_cast<__half*>(a_lo), total);
}

cudaError_t launch_mlp_head_rows(const IstMlpWeights& w, const IstMlpParams& p, const float* h2_scale, const float* h2_inplane,
                                 cudaStream_t stream) {
  const int total = p.B * p.k * kP;
  if (total <= 0) return cudaSuccess;
  return launch_ex(mlp_head_rows_kernel, (total + 7) / 8, 256, 0, stream, 1, false, p, w, h2_scale, h2_inplane, total);
}

cudaError_t launch_ist_mlp(const IstMlpWeights& w, const IstMlpParams& p, cudaStream_t stream) {
  const int total = p.B * p.k * kP;
  if (total <= 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(p.row_count, 0, sizeof(int), stream);
  if (e != cudaSuccess) return e;
  if ((e = launch_ex(mlp_compact_kernel, (total + 255) / 256, 256, 0, stream, 1, false, p, total)) != cudaSuccess) return e;
  const int mtiles = (total + BM - 1) / BM;
  // layer 1 (both heads side by side): [rows,512] x [1024,512]^T -> hidden1 [rows,1024]
  if ((e = launch_ex(mlp_gemm_kernel<true>, dim3(mtiles, 1024 / BN, 1), 256, 0, stream, 1, false, p, w.s_w1, w.s_b1, w.i_w1,
                     w.i_b1, nullptr, 0, 512, p.hidden1, 1024)) != cudaSuccess)
    return e;
  // layer 2 per head: hidden1[:, h*512:+512] x [256,512]^T -> hidden2[:, h*256:+256]
  if ((e = launch_ex(mlp_gemm_kernel<false>, dim3(mtiles, 256 / BN, 2), 256, 0, stream, 1, false, p, w.s_w2, w.s_b2, w.i_w2,
                     w.i_b2, p.hidden1, 1024, 512, p.hidden2, 512)) != cudaSuccess)
    return e;
  return launch_ex(mlp_head_kernel, (total + 7) / 8, 256, 0, stream, 1, false, p, w, total);
}

}  // namespace gp
