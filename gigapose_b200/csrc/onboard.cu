// Row f16: onboarding from real frames with known poses (BOP `onboarding_static`).  A template of the CAD path is seen
// by a camera that looks at the object origin, with the template intrinsics K_t; an onboarding frame is off-axis and
// has its own K_f.  A virtual camera at the frame's centre, rotated by R_v so that its axis passes through the object
// origin, sees the frame through the homography H = K_t R_v K_f^-1, and its view meets the CAD template contract
// exactly (K = K_t, pose [R_v R | (0, 0, |t|)]).  The host (gigapose_b200/onboarding.py) builds R_v and H^-1 in fp64;
// these kernels apply H^-1 per pixel.
//
// Contract:
//  - Pixel centres are at integer coordinates, as csrc/render.cu projects with K: virtual pixel (column c, row r) is
//    the point (c, r) of the virtual image plane and source pixel (column i, row j) is centred at (i, j).
//  - s = H^-1 (c, r, 1)^T in fp64, (x, y) = (s0 / s2, s1 / s2), with the operation order written in `to_source` and no
//    multiply-add contraction (the file is compiled with -fmad=false).  Nearest sampling takes (rint(x), rint(y)),
//    round half to even: on the identity map x lands on an integer up to rounding and never on a tie.
//  - The source lies inside the frame when s2 > 0 (the ray points in front of the source camera) and that nearest
//    pixel is in [0, W) x [0, H); otherwise RGB and mask are 0.
//  - Boxes (gp_recentre_boxes): xyxy with exclusive max of the virtual pixels whose nearest source pixel is inside
//    the frame with a non-zero mask, on the UNBOUNDED virtual grid (negative and beyond-640 x 480 coordinates are
//    kept: a real object at its own distance may not fit the template image, and only the box matters).  The scan
//    region is the source box widened by 1 px, mapped through H; its side is at most GP_RECENTRE_MAX_SIDE.
//  - Crops (gp_recentre_crop): output pixel -> virtual pixel with gp_crop_resize_pad's index arithmetic for the box
//    (as if the virtual image were the box itself: nothing is clipped), virtual pixel -> source through H^-1, RGB
//    bilinear in fp64 over the four nearest pixel centres (indices clamped to the frame), mask nearest; then
//    gp_crop_resize_pad_rle's fused steps: rgb / 255, x mask, (v - CLIP mean) / CLIP std.  out_M is
//    gp_crop_resize_pad's M for the box.
#include <math.h>
#include <stdio.h>

#include "../../include/gigapose_b200.h"
#include "crop_geometry.cuh"
#include "gigapose_kernels.h"

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kGroup = 32;                   // frames per launch; their maps travel by value in the kernel parameters
constexpr int kScanBlocks = 1024;            // blocks per frame of the box scan (grid-stride over the scan region)
constexpr double kMaxCoord = 16777216.0;     // 2^24 px: virtual coordinates stay exact in int32 and fp64 products

struct FrameMaps {
  double hinv[kGroup][9];                    // virtual -> source, row-major
  int scan[kGroup][4];                       // x0, y0, width, height of the scan region (boxes only)
};

// source point of virtual pixel (c, r); false when its ray points behind the source camera (s2 <= 0)
__device__ __forceinline__ bool to_source(const double* h, double c, double r, double& x, double& y) {
  const double sx = h[0] * c + h[1] * r + h[2];
  const double sy = h[3] * c + h[4] * r + h[5];
  const double sw = h[6] * c + h[7] * r + h[8];
  x = sx / sw;
  y = sy / sw;
  return sw > 0.0;
}

// nearest source pixel of virtual pixel (c, r), false outside the frame
__device__ __forceinline__ bool nearest(const double* h, int c, int r, int H, int W, double& x, double& y, int& ix,
                                        int& iy) {
  if (!to_source(h, (double)c, (double)r, x, y)) return false;
  if (!(fabs(x) < kMaxCoord && fabs(y) < kMaxCoord)) return false;
  ix = (int)rint(x);
  iy = (int)rint(y);
  return ix >= 0 && ix < W && iy >= 0 && iy < H;
}

__global__ void __launch_bounds__(kThreads) box_init_kernel(int n, long long* __restrict__ boxes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  boxes[4 * (size_t)i + 0] = LLONG_MAX;
  boxes[4 * (size_t)i + 1] = LLONG_MAX;
  boxes[4 * (size_t)i + 2] = LLONG_MIN;
  boxes[4 * (size_t)i + 3] = LLONG_MIN;
}

__global__ void __launch_bounds__(kThreads)
box_scan_kernel(int H, int W, int frame_base, const uint8_t* __restrict__ masks, FrameMaps fm,
                long long* __restrict__ boxes) {
  const int f = blockIdx.y, frame = frame_base + f;
  const int x0 = fm.scan[f][0], y0 = fm.scan[f][1], sw = fm.scan[f][2], sh = fm.scan[f][3];
  const double* h = fm.hinv[f];
  const uint8_t* m = masks + (size_t)frame * H * W;
  int lo_x = INT_MAX, lo_y = INT_MAX, hi_x = INT_MIN, hi_y = INT_MIN;
  const long long total = (long long)sw * sh;
  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < total; p += (long long)gridDim.x * blockDim.x) {
    const int c = x0 + (int)(p % sw), r = y0 + (int)(p / sw);
    double x, y;
    int ix, iy;
    if (nearest(h, c, r, H, W, x, y, ix, iy) && m[(size_t)iy * W + ix]) {
      lo_x = min(lo_x, c); hi_x = max(hi_x, c);
      lo_y = min(lo_y, r); hi_y = max(hi_y, r);
    }
  }
  __shared__ int red[4][kThreads / 32];
#pragma unroll
  for (int d = 16; d; d >>= 1) {
    lo_x = min(lo_x, __shfl_xor_sync(0xffffffffu, lo_x, d));
    lo_y = min(lo_y, __shfl_xor_sync(0xffffffffu, lo_y, d));
    hi_x = max(hi_x, __shfl_xor_sync(0xffffffffu, hi_x, d));
    hi_y = max(hi_y, __shfl_xor_sync(0xffffffffu, hi_y, d));
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    red[0][warp] = lo_x; red[1][warp] = lo_y; red[2][warp] = hi_x; red[3][warp] = hi_y;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kThreads / 32; ++w) {
      lo_x = min(lo_x, red[0][w]); lo_y = min(lo_y, red[1][w]);
      hi_x = max(hi_x, red[2][w]); hi_y = max(hi_y, red[3][w]);
    }
    if (hi_x >= lo_x) {
      long long* b = boxes + 4 * (size_t)frame;
      atomicMin(b + 0, (long long)lo_x);
      atomicMin(b + 1, (long long)lo_y);
      atomicMax(b + 2, (long long)hi_x + 1);                          // exclusive max
      atomicMax(b + 3, (long long)hi_y + 1);
    }
  }
}

// an empty re-centred mask gets (0, 0, 0, 0)
__global__ void __launch_bounds__(kThreads) box_finish_kernel(int n, long long* __restrict__ boxes) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  long long* b = boxes + 4 * (size_t)i;
  if (b[2] < b[0]) b[0] = b[1] = b[2] = b[3] = 0;
}

__global__ void __launch_bounds__(kThreads)
recentre_crop_kernel(int H, int W, int T, int frame_base, const uint8_t* __restrict__ images,
                     const uint8_t* __restrict__ masks, FrameMaps fm, const long long* __restrict__ boxes,
                     float* __restrict__ out, float* __restrict__ out_mask, float* __restrict__ out_M) {
  constexpr float kMean[3] = {0.48145466f, 0.4578275f, 0.40821073f};  // CLIP (configs/data/transform.yaml:2-7)
  constexpr float kStd[3] = {0.26862954f, 0.26130258f, 0.27577711f};
  __shared__ gp::CropGeom sg;
  __shared__ long long sbox[2];
  const int f = blockIdx.y, frame = frame_base + f;
  if (threadIdx.x == 0) {
    const long long* box = boxes + 4 * (size_t)frame;
    // the crop of gp_crop_resize_pad for a box that lies wholly inside its image: the box itself as the image
    const long long local[4] = {0, 0, box[2] - box[0], box[3] - box[1]};
    const long long bw = max(local[2], 0ll), bh = max(local[3], 0ll);
    sg = gp::crop_geometry(local, (int)min(bh, (long long)INT_MAX), (int)min(bw, (long long)INT_MAX), T);
    sbox[0] = box[0];
    sbox[1] = box[1];
    if (blockIdx.x == 0) gp::write_M(sg, box, out_M + 9 * (size_t)frame);
  }
  __syncthreads();
  const gp::CropGeom g = sg;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= T * T) return;
  const int oy = pix / T, ox = pix - oy * T;
  int row = 0, col = 0;
  bool inside = gp::source_pixel(g, oy, ox, row, col);
  double x = 0.0, y = 0.0;
  int ix = 0, iy = 0;
  if (inside) inside = nearest(fm.hinv[f], (int)(sbox[0] + col), (int)(sbox[1] + row), H, W, x, y, ix, iy);
  const size_t plane = (size_t)H * W;
  float m = 0.f;
  float rgb[3] = {0.f, 0.f, 0.f};
  if (inside) {
    m = masks[(size_t)frame * plane + (size_t)iy * W + ix] ? 1.f : 0.f;
    const double fx0 = floor(x), fy0 = floor(y);
    const double ax = x - fx0, ay = y - fy0;
    const int xa = min(max((int)fx0, 0), W - 1), xb = min(max((int)fx0 + 1, 0), W - 1);
    const int ya = min(max((int)fy0, 0), H - 1), yb = min(max((int)fy0 + 1, 0), H - 1);
    const uint8_t* img = images + (size_t)frame * plane * 3;
    const uint8_t* p00 = img + ((size_t)ya * W + xa) * 3;
    const uint8_t* p01 = img + ((size_t)ya * W + xb) * 3;
    const uint8_t* p10 = img + ((size_t)yb * W + xa) * 3;
    const uint8_t* p11 = img + ((size_t)yb * W + xb) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double top = (1.0 - ax) * (double)p00[c] + ax * (double)p01[c];
      const double bot = (1.0 - ax) * (double)p10[c] + ax * (double)p11[c];
      rgb[c] = (float)((1.0 - ay) * top + ay * bot);
    }
  }
  out_mask[(size_t)frame * T * T + pix] = m;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float v = 0.f;
    if (inside) v = __fmul_rn(__fdiv_rn(rgb[c], 255.f), m);           // rgb / 255.0, x mask: separate roundings
    v = __fdiv_rn(__fsub_rn(v, kMean[c]), kStd[c]);
    out[((size_t)frame * 3 + c) * T * T + pix] = v;
  }
}

bool invert3(const double* a, double* inv) {
  const double c00 = a[4] * a[8] - a[5] * a[7], c01 = a[5] * a[6] - a[3] * a[8], c02 = a[3] * a[7] - a[4] * a[6];
  const double det = a[0] * c00 + a[1] * c01 + a[2] * c02;
  if (!(fabs(det) > 0.0) || !isfinite(det)) return false;
  inv[0] = c00 / det; inv[1] = (a[2] * a[7] - a[1] * a[8]) / det; inv[2] = (a[1] * a[5] - a[2] * a[4]) / det;
  inv[3] = c01 / det; inv[4] = (a[0] * a[8] - a[2] * a[6]) / det; inv[5] = (a[2] * a[3] - a[0] * a[5]) / det;
  inv[6] = c02 / det; inv[7] = (a[1] * a[6] - a[0] * a[7]) / det; inv[8] = (a[0] * a[4] - a[1] * a[3]) / det;
  return true;
}

int check_maps(int n, const double* hinv) {
  for (int i = 0; i < 9 * n; ++i)
    if (!isfinite(hinv[i])) return fail(GP_ERR_INVALID, "frame %d: virtual_to_source holds a non-finite value", i / 9);
  return GP_OK;
}

// scan region of frame i: the source box widened by 1 px, its corners mapped through H = (H^-1)^-1
int scan_region(int i, const double* hinv, const int64_t* src_box, int* scan) {
  double h[9];
  if (!invert3(hinv, h)) return fail(GP_ERR_INVALID, "frame %d: virtual_to_source is singular", i);
  const double xs[2] = {(double)src_box[0] - 1.0, (double)src_box[2]};
  const double ys[2] = {(double)src_box[1] - 1.0, (double)src_box[3]};
  double lo_x = INFINITY, lo_y = INFINITY, hi_x = -INFINITY, hi_y = -INFINITY;
  for (double x : xs)
    for (double y : ys) {
      const double w = h[6] * x + h[7] * y + h[8];
      if (!(w > 0.0)) return fail(GP_ERR_INVALID, "frame %d: the mask box reaches the virtual camera's horizon", i);
      const double u = (h[0] * x + h[1] * y + h[2]) / w, v = (h[3] * x + h[4] * y + h[5]) / w;
      lo_x = fmin(lo_x, u); hi_x = fmax(hi_x, u);
      lo_y = fmin(lo_y, v); hi_y = fmax(hi_y, v);
    }
  lo_x = floor(lo_x) - 1.0; lo_y = floor(lo_y) - 1.0;
  hi_x = ceil(hi_x) + 1.0; hi_y = ceil(hi_y) + 1.0;
  if (!(fabs(lo_x) < kMaxCoord && fabs(lo_y) < kMaxCoord && fabs(hi_x) < kMaxCoord && fabs(hi_y) < kMaxCoord))
    return fail(GP_ERR_INVALID, "frame %d: the re-centred mask lies beyond 2^24 px of the virtual principal point", i);
  const double sw = hi_x - lo_x + 1.0, sh = hi_y - lo_y + 1.0;
  if (sw > GP_RECENTRE_MAX_SIDE || sh > GP_RECENTRE_MAX_SIDE)
    return fail(GP_ERR_INVALID, "frame %d: re-centred scan region %.0f x %.0f px exceeds GP_RECENTRE_MAX_SIDE = %d", i,
                sw, sh, GP_RECENTRE_MAX_SIDE);
  scan[0] = (int)lo_x; scan[1] = (int)lo_y; scan[2] = (int)sw; scan[3] = (int)sh;
  return GP_OK;
}

}  // namespace

extern "C" int gp_recentre_boxes(int n, int height, int width, const uint8_t* masks, const double* virtual_to_source,
                                 const int64_t* src_boxes, int64_t* out_boxes, void* stream) {
  if (n < 0 || height < 1 || width < 1) return fail(GP_ERR_INVALID, "bad shape");
  if (n == 0) return GP_OK;
  if (!masks || !virtual_to_source || !src_boxes || !out_boxes) return fail(GP_ERR_INVALID, "null argument");
  if (const int rc = check_maps(n, virtual_to_source)) return rc;
  for (int i = 0; i < n; ++i) {
    const int64_t* b = src_boxes + 4 * (size_t)i;
    if (b[2] > b[0] && (b[0] < 0 || b[1] < 0 || b[2] > width || b[3] > height || b[3] <= b[1]))
      return fail(GP_ERR_INVALID, "frame %d: source box (%lld, %lld, %lld, %lld) outside the %d x %d frame", i,
                  (long long)b[0], (long long)b[1], (long long)b[2], (long long)b[3], width, height);
  }
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long* boxes = reinterpret_cast<long long*>(out_boxes);
  GP_CUDA(gp::launch_ex(box_init_kernel, (n + kThreads - 1) / kThreads, kThreads, 0, s, 1, false, n, boxes));
  for (int f0 = 0; f0 < n; f0 += kGroup) {
    const int g = min(kGroup, n - f0);
    FrameMaps fm = {};
    long long largest = 0;
    for (int f = 0; f < g; ++f) {
      const int64_t* b = src_boxes + 4 * (size_t)(f0 + f);
      for (int k = 0; k < 9; ++k) fm.hinv[f][k] = virtual_to_source[9 * (size_t)(f0 + f) + k];
      if (b[2] <= b[0]) continue;                                     // empty mask: nothing to scan
      if (const int rc = scan_region(f0 + f, fm.hinv[f], b, fm.scan[f])) return rc;
      largest = max(largest, (long long)fm.scan[f][2] * fm.scan[f][3]);
    }
    if (!largest) continue;
    const int blocks = (int)min((largest + kThreads - 1) / kThreads, (long long)kScanBlocks);
    GP_CUDA(gp::launch_ex(box_scan_kernel, dim3(blocks, g), kThreads, 0, s, 1, false, height, width, f0, masks, fm, boxes));
  }
  GP_CUDA(gp::launch_ex(box_finish_kernel, (n + kThreads - 1) / kThreads, kThreads, 0, s, 1, false, n, boxes));
  return GP_OK;
}

extern "C" int gp_recentre_crop(int n, int height, int width, int target_size, const uint8_t* images,
                                const uint8_t* masks, const double* virtual_to_source, const int64_t* boxes,
                                float* out_images, float* out_mask, float* out_M, void* stream) {
  if (n < 0 || height < 1 || width < 1) return fail(GP_ERR_INVALID, "bad shape");
  if (target_size < 128 || target_size > 4096)
    return fail(GP_ERR_INVALID, "target_size %d outside [128, 4096] (smaller outputs take a different ATen path)", target_size);
  if (n == 0) return GP_OK;
  if (!images || !masks || !virtual_to_source || !boxes || !out_images || !out_mask || !out_M)
    return fail(GP_ERR_INVALID, "null argument");
  if (const int rc = check_maps(n, virtual_to_source)) return rc;
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  for (int f0 = 0; f0 < n; f0 += kGroup) {
    const int g = min(kGroup, n - f0);
    FrameMaps fm = {};
    for (int f = 0; f < g; ++f)
      for (int k = 0; k < 9; ++k) fm.hinv[f][k] = virtual_to_source[9 * (size_t)(f0 + f) + k];
    const dim3 grid((target_size * target_size + kThreads - 1) / kThreads, g);
    GP_CUDA(gp::launch_ex(recentre_crop_kernel, grid, kThreads, 0, s, 1, false, height, width, target_size, f0, images,
                          masks, fm, reinterpret_cast<const long long*>(boxes), out_images, out_mask, out_M));
  }
  return GP_OK;
}
