// Row f3 of SURVEY.md §8: query pre-processing on the GPU.  `CropResizePad.__call__` (reference src/utils/crop.py:16-61:
// crop the detection box, nearest-neighbour resize so that the longer box side becomes `target`, centred zero padding
// to target x target, nearest resize to exactly target x target, and the 3x3 matrix M of that map) fused with the
// element-wise steps around it in the dataloader (`process_real`, dataloader/train.py:80-123: /255, x mask; CLIP
// mean/std normalisation, configs/data/transform.yaml:2-7).  The reference does this per detection in a python loop on
// the CPU; here one thread produces one output pixel (all channels) by composing the index maps -- a pure gather.
//
// Index arithmetic follows ATen's CPU nearest kernels: out = floor(in * scale) in double, src = min(floorf(dst *
// float(1 / scale)), in - 1) for the first resize (with the identity / dst >> 1 special cases of the small-output kernel
// when out_h + out_w <= 128), src = min(floorf(dst * (float(in) / out)), in - 1) for the second, whose output
// (2 * target > 128) always takes the plain path.
#include "../../include/gigapose_b200.h"
#include "crop_geometry.cuh"
#include "gigapose_kernels.h"

using gp::fail;

using gp::CropGeom;
using gp::crop_geometry;
using gp::source_pixel;
using gp::write_M;

namespace {

__global__ void __launch_bounds__(256)
crop_resize_pad_kernel(int C, int H, int W, int T, const float* __restrict__ images, const int* __restrict__ image_index,
                       const long long* __restrict__ boxes, const float* __restrict__ mask, float in_div,
                       const float* __restrict__ post_sub, const float* __restrict__ post_div, float* __restrict__ out,
                       float* __restrict__ out_mask, float* __restrict__ out_M) {
  __shared__ CropGeom sg;
  const int det = blockIdx.y;
  if (threadIdx.x == 0) {
    sg = crop_geometry(boxes + 4 * (size_t)det, H, W, T);
    if (blockIdx.x == 0 && out_M) write_M(sg, boxes + 4 * (size_t)det, out_M + 9 * (size_t)det);
  }
  __syncthreads();
  const CropGeom g = sg;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= T * T) return;
  const int oy = pix / T, ox = pix - oy * T;
  int row = 0, col = 0;
  const bool inside = source_pixel(g, oy, ox, row, col);
  const size_t src = inside ? (size_t)row * W + col : 0;
  const size_t plane = (size_t)H * W;
  const size_t img = image_index ? (size_t)image_index[det] : (size_t)det;
  float m = 1.f;
  if (mask) {
    m = inside ? mask[(size_t)det * plane + src] : 0.f;
    if (out_mask) out_mask[(size_t)det * T * T + pix] = m;
  }
  for (int c = 0; c < C; ++c) {
    float v = 0.f;                                                     // padding is zero BEFORE the normalisation
    if (inside) {
      v = images[(img * C + c) * plane + src];
      if (in_div != 1.f) v = __fdiv_rn(v, in_div);                     // individually rounded, never contracted into
      if (mask) v = __fmul_rn(v, m);                                   // FMAs: the reference runs them as separate ops
    }
    if (post_sub) v = __fsub_rn(v, post_sub[c]);
    if (post_div) v = __fdiv_rn(v, post_div[c]);
    out[((size_t)det * C + c) * T * T + pix] = v;
  }
}

// ---- gp_crop_resize_pad_rle: the same crop with the mask read from its COCO run-length encoding ---------------------
// Detections go to the device in groups of kRleGroup, their run offsets by value (host memory, no device copy).
constexpr int kRleGroup = 256;
struct RleOffsets {
  long long off[kRleGroup + 1];       // detection base + i owns counts / ends [off[i], off[i + 1])
};

// ends[k] = counts[off] + ... + counts[k] over each detection's runs: one CTA per detection, 4 runs per thread per tile.
__global__ void __launch_bounds__(256)
rle_scan_kernel(const int32_t* __restrict__ counts, RleOffsets ro, long long* __restrict__ ends) {
  __shared__ long long warp_sum[8];
  __shared__ long long carry_s;
  const long long r0 = ro.off[blockIdx.x], r1 = ro.off[blockIdx.x + 1];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long carry = 0;
  for (long long t0 = r0; t0 < r1; t0 += 4 * 256) {
    const long long i0 = t0 + 4 * threadIdx.x;
    long long v[4], s = 0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      v[j] = i0 + j < r1 ? (long long)counts[i0 + j] : 0;
      s += v[j];
      v[j] = s;                                                        // inclusive within the thread
    }
    long long x = s;                                                   // inclusive over the warp
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const long long y = __shfl_up_sync(0xffffffffu, x, d);
      if (lane >= d) x += y;
    }
    if (lane == 31) warp_sum[warp] = x;
    __syncthreads();
    long long before = carry + x - s;                                  // everything before this thread's first run
    for (int w = 0; w < warp; ++w) before += warp_sum[w];
#pragma unroll
    for (int j = 0; j < 4; ++j)
      if (i0 + j < r1) ends[i0 + j] = before + v[j];
    if (threadIdx.x == 255) carry_s = before + s;
    __syncthreads();
    carry = carry_s;
  }
}

__device__ __forceinline__ float rle_value(const long long* __restrict__ ends, long long r0, long long r1, long long p) {
  return gp::rle_bit(ends, r0, r1, p) ? 1.f : 0.f;
}

__global__ void __launch_bounds__(256)
crop_resize_pad_rle_kernel(int H, int W, int T, int det_base, const uint8_t* __restrict__ images,
                           const int* __restrict__ image_index, const long long* __restrict__ boxes, RleOffsets ro,
                           const long long* __restrict__ ends, float* __restrict__ out, float* __restrict__ out_mask,
                           float* __restrict__ out_M) {
  constexpr float kMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};  // CLIP (configs/data/transform.yaml:2-7)
  constexpr float kStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};
  __shared__ CropGeom sg;
  const int det = det_base + blockIdx.y;
  if (threadIdx.x == 0) {
    sg = crop_geometry(boxes + 4 * (size_t)det, H, W, T);
    if (blockIdx.x == 0) write_M(sg, boxes + 4 * (size_t)det, out_M + 9 * (size_t)det);
  }
  __syncthreads();
  const CropGeom g = sg;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= T * T) return;
  const int oy = pix / T, ox = pix - oy * T;
  int row = 0, col = 0;
  const bool inside = source_pixel(g, oy, ox, row, col);
  float m = 0.f;
  const uint8_t* px = nullptr;
  if (inside) {
    m = rle_value(ends, ro.off[blockIdx.y], ro.off[blockIdx.y + 1], (long long)col * H + row);   // column-major
    px = images + (((size_t)image_index[det] * H + row) * W + col) * 3;                           // HWC
  }
  out_mask[(size_t)det * T * T + pix] = m;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = 0.f;
    if (inside) v = __fmul_rn(__fdiv_rn((float)px[c], 255.f), m);     // rgb / 255.0, x mask: separate roundings
    v = __fdiv_rn(__fsub_rn(v, kMean[c]), kStd[c]);
    out[((size_t)det * 3 + c) * T * T + pix] = v;
  }
}

}  // namespace

cudaError_t gp::launch_rle_scan(int n, const int32_t* counts, const int64_t* offsets, long long* ends, cudaStream_t s) {
  for (int d0 = 0; d0 < n; d0 += kRleGroup) {
    const int g = min(kRleGroup, n - d0);
    RleOffsets ro;
    for (int i = 0; i <= g; ++i) ro.off[i] = offsets[d0 + i];
    if (const cudaError_t e = gp::launch_ex(rle_scan_kernel, dim3(g), 256, 0, s, 1, false, counts, ro, ends)) return e;
  }
  return cudaSuccess;
}

extern "C" int gp_crop_resize_pad(int n, int channels, int height, int width, int target_size, const float* images,
                                  const int32_t* image_index, const int64_t* xyxy_boxes, const float* mask, float in_div,
                                  const float* post_sub, const float* post_div, float* out_images, float* out_mask,
                                  float* out_M, void* stream) {
  if (n < 0 || channels < 1 || height < 1 || width < 1) return fail(GP_ERR_INVALID, "bad shape");
  if (target_size < 128 || target_size > 4096)
    return fail(GP_ERR_INVALID, "target_size %d outside [128, 4096] (smaller outputs take a different ATen path)", target_size);
  if (!images || !xyxy_boxes || !out_images) return fail(GP_ERR_INVALID, "null argument");
  if (out_mask && !mask) return fail(GP_ERR_INVALID, "out_mask needs mask");
  if (!(in_div > 0.f)) return fail(GP_ERR_INVALID, "in_div must be positive");
  if (n == 0) return GP_OK;
  const dim3 grid((target_size * target_size + 255) / 256, n);
  GP_CUDA(gp::launch_ex(crop_resize_pad_kernel, grid, 256, 0, static_cast<cudaStream_t>(stream), 1, false, channels, height,
                        width, target_size, images, image_index, reinterpret_cast<const long long*>(xyxy_boxes), mask,
                        in_div, post_sub, post_div, out_images, out_mask, out_M));
  return GP_OK;
}

extern "C" int gp_crop_resize_pad_rle(int n, int height, int width, int target_size, const uint8_t* images,
                                      const int32_t* image_index, const int64_t* xyxy_boxes, const int32_t* counts,
                                      const int64_t* offsets, int64_t* ends, float* out_images, float* out_mask,
                                      float* out_M, void* stream) {
  if (n < 0 || height < 1 || width < 1) return fail(GP_ERR_INVALID, "bad shape");
  if (target_size < 128 || target_size > 4096)
    return fail(GP_ERR_INVALID, "target_size %d outside [128, 4096] (smaller outputs take a different ATen path)", target_size);
  if (!images || !image_index || !xyxy_boxes || !offsets || !out_images || !out_mask || !out_M)
    return fail(GP_ERR_INVALID, "null argument");
  if (offsets[0] < 0) return fail(GP_ERR_INVALID, "offsets[0] = %lld is negative", (long long)offsets[0]);
  for (int i = 0; i < n; ++i)
    if (offsets[i + 1] < offsets[i])
      return fail(GP_ERR_INVALID, "offsets decrease at detection %d (%lld -> %lld)", i, (long long)offsets[i],
                  (long long)offsets[i + 1]);
  if (offsets[n] > offsets[0] && (!counts || !ends)) return fail(GP_ERR_INVALID, "null counts / ends");
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int d0 = 0; d0 < n; d0 += kRleGroup) {
    const int g = min(kRleGroup, n - d0);
    RleOffsets ro;
    for (int i = 0; i <= g; ++i) ro.off[i] = offsets[d0 + i];
    GP_CUDA(gp::launch_ex(rle_scan_kernel, dim3(g), 256, 0, s, 1, false, counts, ro, reinterpret_cast<long long*>(ends)));
    const dim3 grid((target_size * target_size + 255) / 256, g);
    GP_CUDA(gp::launch_ex(crop_resize_pad_rle_kernel, grid, 256, 0, s, 1, false, height, width, target_size, d0, images,
                          image_index, reinterpret_cast<const long long*>(xyxy_boxes), ro,
                          reinterpret_cast<const long long*>(ends), out_images, out_mask, out_M));
  }
  return GP_OK;
}
