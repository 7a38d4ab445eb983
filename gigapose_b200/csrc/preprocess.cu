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
#include "gigapose_kernels.h"

using gp::fail;

namespace {

struct CropGeom {
  int x1, y1, ch, cw;        // crop origin and size after clipping to the image
  int rh, rw;                // size after the first resize
  int pad_top, pad_left, ph, pw;
  float inv1;                // float(1 / scale)
  float inv_h2, inv_w2;      // float(ph) / target, float(pw) / target
  float scale;
};

__device__ CropGeom crop_geometry(const long long* box, int H, int W, int T) {
  CropGeom g;
  const long long bx1 = max(box[0], 0ll), by1 = max(box[1], 0ll), bx2 = box[2], by2 = box[3];
  g.x1 = (int)min(bx1, (long long)W); g.y1 = (int)min(by1, (long long)H);
  g.cw = max((int)min(bx2, (long long)W) - g.x1, 0);
  g.ch = max((int)min(by2, (long long)H) - g.y1, 0);
  const long long side = max(box[2] - box[0], box[3] - box[1]);        // the un-clipped box decides the scale (crop.py:19-20)
  // `target / sizes.max()` on an integer tensor is `sizes.reciprocal() * target` in float32 (Tensor.__rtruediv__): two
  // roundings, not one division
  g.scale = __fmul_rn(__frcp_rn((float)side), (float)T);
  const double sd = (double)g.scale;
  g.rh = (int)floor((double)g.ch * sd);
  g.rw = (int)floor((double)g.cw * sd);
  g.inv1 = (float)(1.0 / sd);
  g.pad_top = g.pad_left = 0;
  g.ph = g.rh; g.pw = g.rw;
  if (g.rw != g.rh) {                                                  // crop.py:37-46
    g.pad_top = (T - g.rh) / 2;                                        // sizes never exceed T: plain division == floor
    const int pad_bottom = max(T - g.rh - g.pad_top, 0);
    g.pad_left = max((T - g.rw) / 2, 0);
    const int pad_right = T - g.rw - g.pad_left;
    g.ph = g.rh + g.pad_top + pad_bottom;
    g.pw = g.rw + g.pad_left + pad_right;
  }
  g.inv_h2 = (float)g.ph / (float)T;
  g.inv_w2 = (float)g.pw / (float)T;
  return g;
}

__global__ void __launch_bounds__(256)
crop_resize_pad_kernel(int C, int H, int W, int T, const float* __restrict__ images, const int* __restrict__ image_index,
                       const long long* __restrict__ boxes, const float* __restrict__ mask, float in_div,
                       const float* __restrict__ post_sub, const float* __restrict__ post_div, float* __restrict__ out,
                       float* __restrict__ out_mask, float* __restrict__ out_M) {
  __shared__ CropGeom sg;
  const int det = blockIdx.y;
  if (threadIdx.x == 0) {
    sg = crop_geometry(boxes + 4 * (size_t)det, H, W, T);
    if (blockIdx.x == 0 && out_M) {                                    // M = M_resize_pad @ M_crop (crop.py:28-48)
      float* M = out_M + 9 * (size_t)det;
      const float s = sg.scale;
      const bool padded = sg.rw != sg.rh;
      M[0] = s; M[1] = 0.f; M[2] = fmaf(s, -(float)boxes[4 * (size_t)det + 0], padded ? (float)sg.pad_left : 0.f);
      M[3] = 0.f; M[4] = s; M[5] = fmaf(s, -(float)boxes[4 * (size_t)det + 1], padded ? (float)sg.pad_top : 0.f);
      M[6] = 0.f; M[7] = 0.f; M[8] = 1.f;
    }
  }
  __syncthreads();
  const CropGeom g = sg;
  const int pix = blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= T * T) return;
  const int oy = pix / T, ox = pix - oy * T;
  // second resize (target x target <- padded), then un-pad, then first resize (resized <- crop), then un-crop
  int pr = min((int)floorf((float)oy * g.inv_h2), g.ph - 1) - g.pad_top;
  int pc = min((int)floorf((float)ox * g.inv_w2), g.pw - 1) - g.pad_left;
  const bool inside = pr >= 0 && pr < g.rh && pc >= 0 && pc < g.rw;
  size_t src = 0;
  if (inside) {
    // ATen routes outputs with out_h + out_w <= 128 (a heavily clipped box) to a kernel whose index function keeps an
    // unchanged size as the identity and an exactly doubled size as dst >> 1 instead of the float arithmetic
    const bool small = g.rh + g.rw <= 128;
    int lr, lc;
    if (small && g.rh == g.ch) lr = pr;
    else if (small && g.rh == 2 * g.ch) lr = pr >> 1;
    else lr = min((int)floorf((float)pr * g.inv1), g.ch - 1);
    if (small && g.rw == g.cw) lc = pc;
    else if (small && g.rw == 2 * g.cw) lc = pc >> 1;
    else lc = min((int)floorf((float)pc * g.inv1), g.cw - 1);
    src = (size_t)(g.y1 + lr) * W + (g.x1 + lc);
  }
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

}  // namespace

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
