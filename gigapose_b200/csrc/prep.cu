// Descriptor / mask preparation kernels (rows a2-a4 of SURVEY.md §8):
//  * split_descriptors: L2-normalise patch descriptors (ae_net.py:69 and again matching.py:224/229 -- the reference
//    normalises twice and the second pass changes bits) and store them as bf16 hi/lo planes, patch-major and
//    K-contiguous, the layout the TMA/wgmma similarity kernel consumes;
//  * sample_mask16: nearest 224->16 mask sampling (matching.py:222,227; F.interpolate default = nearest);
//  * transpose_cp: channel-major [n,C,256] -> patch-major [n,256,C] (IST features for the gather of ist_net.py:98-99).
// All HBM-bound byte movers: coalesced, vectorised where the layout allows.
#include "gigapose_kernels.h"
#include <cuda_bf16.h>

namespace gp {

namespace {

__device__ __forceinline__ float block_sum_256(float v, float* s_red) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) s_red[warp] = v;
  __syncthreads();
  float t = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) t += s_red[w];
  return t;
}

// one CTA (256 threads) per descriptor row; C <= 256 * kMaxPerThread
constexpr int kMaxPerThread = 8;

__global__ void __launch_bounds__(256)
split_descriptors_kernel(const float* __restrict__ x, long long n_rows, int C, int rows_per_img, long long img_stride,
                         long long row_stride, long long chan_stride, int norm_passes, int tiled,
                         __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo, float* __restrict__ normalized_out) {
  __shared__ float s_red[8];
  const long long r = blockIdx.x;
  if (r >= n_rows) return;
  const float* src = x + (r / rows_per_img) * img_stride + (r % rows_per_img) * row_stride;
  float v[kMaxPerThread];
  const int per = (C + 255) / 256;
#pragma unroll
  for (int i = 0; i < kMaxPerThread; ++i) {
    const int c = threadIdx.x + i * 256;
    v[i] = (i < per && c < C) ? src[(long long)c * chan_stride] : 0.f;
  }
  for (int pass = 0; pass < norm_passes; ++pass) {
    float ss = 0.f;
#pragma unroll
    for (int i = 0; i < kMaxPerThread; ++i) ss += v[i] * v[i];
    const float nrm = fmaxf(sqrtf(block_sum_256(ss, s_red)), 1e-12f);   // F.normalize: x / max(||x||, eps)
#pragma unroll
    for (int i = 0; i < kMaxPerThread; ++i) v[i] = v[i] / nrm;
  }
#pragma unroll
  for (int i = 0; i < kMaxPerThread; ++i) {
    const int c = threadIdx.x + i * 256;
    if (i < per && c < C) {
      const __nv_bfloat16 h = __float2bfloat16_rn(v[i]);
      const __nv_bfloat16 l = __float2bfloat16_rn(v[i] - __bfloat162float(h));
      // k-block-tiled planes: [image][c / 32][patch][c % 32] -- the 256 x 32 box the similarity kernel's TMA fetches
      // per K-block is one contiguous 16 KB slab (streams from HBM at full page locality when nothing is shared)
      const size_t o = tiled ? ((((size_t)(r / rows_per_img) * (C / 32) + (c >> 5)) * rows_per_img + (r % rows_per_img)) << 5) + (c & 31)
                             : (size_t)r * C + c;
      if (hi) { hi[o] = h; lo[o] = l; }
      if (normalized_out) normalized_out[r * C + c] = v[i];
    }
  }
}

__global__ void sample_mask16_kernel(const float* __restrict__ mask, long long n, int H, int W, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n * 256) return;
  const long long img = i >> 8;
  const int p = (int)(i & 255), py = p >> 4, px = p & 15;
  // PyTorch nearest: src = floor(dst * in / out) computed in float
  const int sy = min((int)floorf(py * ((float)H / 16.0f)), H - 1);
  const int sx = min((int)floorf(px * ((float)W / 16.0f)), W - 1);
  out[i] = mask[(img * H + sy) * W + sx];
}

// [n, C, 256] -> [n, 256, C] through a 32x32 smem tile
__global__ void transpose_cp_kernel(const float* __restrict__ in, int C, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const long long img = blockIdx.z;
  const int c0 = blockIdx.y * 32, p0 = blockIdx.x * 32;
  const float* src = in + img * (long long)C * 256;
  float* dst = out + img * (long long)C * 256;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    tile[i][threadIdx.x] = (c < C) ? src[(long long)c * 256 + p0 + threadIdx.x] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + threadIdx.x;
    if (c < C) dst[(long long)(p0 + i) * C + c] = tile[threadIdx.x][i];
  }
}

// perm = stable order of the queries by object id (rank by counting; B is at most a few hundred)
// also writes the clamped copy of the object ids the other kernels index the bank with
__global__ void object_order_kernel(const int* __restrict__ q_obj, int B, int num_objects, int* __restrict__ q_obj_out,
                                    int* __restrict__ perm) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B; i += gridDim.x * blockDim.x) {
    const int mine = min(max(q_obj[i], 0), num_objects - 1);
    int rank = 0;
    for (int j = 0; j < B; ++j) {
      const int o = min(max(q_obj[j], 0), num_objects - 1);
      rank += (o < mine || (o == mine && j < i)) ? 1 : 0;
    }
    perm[rank] = i;
    q_obj_out[i] = mine;
  }
}

}  // namespace

cudaError_t launch_object_order(const int* q_obj, int B, int num_objects, int* q_obj_out, int* perm, cudaStream_t stream) {
  if (B <= 0) return cudaSuccess;
  return launch_ex(object_order_kernel, (B + 127) / 128, 128, 0, stream, 1, false, q_obj, B, num_objects, q_obj_out, perm);
}

cudaError_t launch_split_descriptors(const float* x, long long n_rows, int C, int rows_per_img, long long img_stride,
                                     long long row_stride, long long chan_stride, int norm_passes, int tiled, uint16_t* hi,
                                     uint16_t* lo, float* normalized_out, cudaStream_t stream) {
  if (n_rows <= 0) return cudaSuccess;
  if (C > 256 * kMaxPerThread) return cudaErrorInvalidValue;
  return launch_ex(split_descriptors_kernel, (unsigned)n_rows, 256, 0, stream, 1, false, x, n_rows, C, rows_per_img, img_stride,
                   row_stride, chan_stride, norm_passes, tiled, reinterpret_cast<__nv_bfloat16*>(hi),
                   reinterpret_cast<__nv_bfloat16*>(lo), normalized_out);
}

cudaError_t launch_sample_mask16(const float* mask, long long n, int H, int W, float* out, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const long long total = n * 256;
  return launch_ex(sample_mask16_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, 1, false, mask, n, H, W, out);
}

cudaError_t launch_transpose_cp(const float* in, long long n, int C, float* out, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  for (long long i0 = 0; i0 < n; i0 += 32768) {          // gridDim.z limit
    const long long cnt = (n - i0 < 32768) ? (n - i0) : 32768;
    dim3 grid(256 / 32, (C + 31) / 32, (unsigned)cnt), block(32, 8);
    cudaError_t e = launch_ex(transpose_cp_kernel, grid, block, 0, stream, 1, false, in + i0 * C * 256, C, out + i0 * C * 256);
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

}  // namespace gp
