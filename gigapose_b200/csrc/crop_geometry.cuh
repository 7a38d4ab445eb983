// The index arithmetic of gp_crop_resize_pad (csrc/preprocess.cu), shared with the onboarding re-centring crop
// (csrc/onboard.cu) so that both map an output pixel to the same box pixel.  Not installed.
#pragma once
#include <cuda_runtime.h>

namespace gp {

struct CropGeom {
  int x1, y1, ch, cw;        // crop origin and size after clipping to the image
  int rh, rw;                // size after the first resize
  int pad_top, pad_left, ph, pw;
  float inv1;                // float(1 / scale)
  float inv_h2, inv_w2;      // float(ph) / target, float(pw) / target
  float scale;
};

inline __device__ CropGeom crop_geometry(const long long* box, int H, int W, int T) {
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

// M = M_resize_pad @ M_crop (crop.py:28-48)
inline __device__ void write_M(const CropGeom& g, const long long* box, float* M) {
  const float s = g.scale;
  const bool padded = g.rw != g.rh;
  M[0] = s; M[1] = 0.f; M[2] = fmaf(s, -(float)box[0], padded ? (float)g.pad_left : 0.f);
  M[3] = 0.f; M[4] = s; M[5] = fmaf(s, -(float)box[1], padded ? (float)g.pad_top : 0.f);
  M[6] = 0.f; M[7] = 0.f; M[8] = 1.f;
}

// Source pixel (row, col) of output pixel (oy, ox), or false where the output is padding: the second resize (target x
// target <- padded), then un-pad, then the first resize (resized <- crop), then un-crop.
inline __device__ bool source_pixel(const CropGeom& g, int oy, int ox, int& row, int& col) {
  const int pr = min((int)floorf((float)oy * g.inv_h2), g.ph - 1) - g.pad_top;
  const int pc = min((int)floorf((float)ox * g.inv_w2), g.pw - 1) - g.pad_left;
  if (!(pr >= 0 && pr < g.rh && pc >= 0 && pc < g.rw)) return false;
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
  row = g.y1 + lr;
  col = g.x1 + lc;
  return true;
}

}  // namespace gp
