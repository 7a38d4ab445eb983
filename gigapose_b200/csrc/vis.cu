// Row f14: the reference's diagnostic images on the GPU.  src/scripts/vis_bop_results.py draws, for each target image,
// the ground truth and each method's estimates over a grey copy of the image with their contours (mask_background,
// draw_contour) and a heat map of the per-vertex error of each estimate (set_texture_visii); GigaPose.vis_retrieval
// (src/models/gigaPose.py:451-479) draws each retrieved template warped by the predicted affine M onto the query crop
// (src/libVis/torch.py::plot_Kabsch).  Their hot paths are the four entry points below; the meshes are rendered by
// gp_render_templates.  Every entry needs no handle, takes caller-owned device memory and an explicit stream, and
// launches through gp::launch_ex.
//
// Contract (what tests/test_gpu_vis.py pins against oracle/vis_port.py bit for bit, and against the cv2 4.13, PIL 12 and
// scipy fixtures of oracle/make_golden_vis.py):
//  Grey.  gray(r, g, b) = (9798 r + 19235 g + 3735 b + 2^14) >> 15 on u8 values, cv2's 8-bit COLOR_RGB2GRAY; GRAY2RGB
//    repeats it.  (The 14-bit form (4899 r + 9617 g + 1868 b + 2^13) >> 14 differs from cv2 4.13 on 0.26 % of the 2^24
//    colours; the 15-bit form equals it on all of them.)
//  Boundary edge of a mask: a mask pixel with a 4-neighbour outside the mask or outside the image.  It stands in for
//    skimage.feature.canny, which the reference uses; the two are not compared (skimage is not a dependency).
//  gp_vis_vertex_errors: add_kernel<true> of csrc/bop_eval.cu (the comment above add_kernel states the arithmetic).  Per
//    (estimate, ground truth) pair, value j is the ADD distance |P_est x_j - P_gt x_j| of vertex j, or with the pair's
//    symmetric flag its ADD-S distance min_i |P_gt x_j - P_est x_i| (the min on the squared terms' float bits, then one
//    sqrt): spatial.distance_matrix(gt, pred).min(axis=1) of set_texture_visii.  The fp64 sums of gp_bop_add are sums
//    of exactly these values.
//  gp_vis_heat_colors: per pair, d = (double)v / (double)max_distance over the pair's values v, with max_distance (and
//    0 for a symmetric pair) appended as set_texture_visii appends them; x = (d - min d) / (max d - min d) in fp64
//    (trimesh.visual.color.interpolate; for a non-symmetric pair the range starts at its smallest value, not at 0);
//    colour = kTurbo[min(floor(256 x), 255)] (matplotlib's Colormap.__call__), written as f32 c / 255.f.  A pair with a
//    NaN value, or with max d = min d, gets (0, 0, 0) for every vertex (matplotlib's "bad" colour: numpy's min / max
//    propagate the NaN).  max_distance is in the unit of the values: the reference's 10 is in its scene unit, the mesh
//    scaled by 0.1 from mm (add_obj / set_object_pose), so it is 100 mm.  kTurbo is
//    cv2.applyColorMap(np.arange(256, dtype=np.uint8), cv2.COLORMAP_TURBO) in RGB order; whether it equals
//    round(255 x matplotlib's _turbo_data) is not verified (matplotlib is not a dependency).
//  gp_vis_overlay, one thread per pixel: out = the background (the image's grey, or 0 without an image), then for each
//    layer l in order: where alpha_l > 0 (the mask onboarding uses) the render's RGB, rint(255 c) (exact: the renderer
//    resolves to k / 255); then, with outline colours, the layer's contour pixels take colour_l.  The contour is the
//    boundary edge of the mask dilated by scipy.ndimage.binary_dilation(edge, np.ones((2, 2))): pixel (y, x) is on it
//    when any of (y, x), (y, x + 1), (y + 1, x), (y + 1, x + 1) is an edge pixel.  A layer is skipped outside its box
//    grown by one pixel up and left (no mask pixel lies outside the box).
//  gp_vis_kabsch, plot_Kabsch for 224 x 224 crops, one thread per pixel of a 16 x 16 tile:
//    unnormalise: convert_tensor_to_image, torchvision's Normalize with the reference's inverse ImageNet statistics
//      (mean -m_c / s_c, std 1 / s_c, each a double rounded to f32) as one fp32 sub and one fp32 div, then x 255 in
//      fp32, then np.uint8: truncation to int32 (0 outside the int32 range or for NaN), low 8 bits.  Masks: x 255, the
//      same cast.  The crops are CLIP-normalised and the reference unnormalises them with ImageNet's statistics; that
//      is kept.
//    query: grey.  template: RGBA (mask as alpha) warped by M[:2] as cv2.warpAffine(src, M[:2], (224, 224)) does with
//      INTER_LINEAR and BORDER_CONSTANT 0: M inverted in fp64 (D = 1 / (M00 M11 - M01 M10), 0 for a singular M), then per
//      destination pixel X = (rint((iM01 y + iM02) 1024) + 16 + rint(iM00 x 1024)) >> 5 (likewise Y), the source
//      pixel (X >> 5, Y >> 5) saturated to int16 and the weights of the fractions fx = X & 31, fy = Y & 31:
//      w00 = 32 (32 - fx)(32 - fy), w01 = 32 fx (32 - fy), w10 = 32 (32 - fx) fy, w11 = 32 fx fy (cv2's float
//      weights times 2^15, exact integers); out = (sum w s + 2^14) >> 15, taps outside the crop reading 0.
//    paste: PIL's Image.paste(rgb, (0, 0), alpha): out = DIV255(grey (255 - a) + w a), DIV255(t) = ((t + 128) >> 8 +
//      t + 128) >> 8.
//    edges: create_edge_from_mask, the boundary edge of DIV255(a a) > 0 (the mask pasted onto black through itself)
//      dilated by a 3 x 3 square; red (255, 0, 0) on the warped alpha's edge, then green (0, 255, 0) on the query
//      mask's.  The reference's keypoint panel (cv2.drawMatchesKnn with random colours) is not drawn.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kCrop = GP_VIS_CROP;
constexpr int kTile = 16;
constexpr int kHalo = kTile + 4;                         // the tile and the 2-pixel ring its edges and dilation read

__constant__ uint8_t kTurbo[256 * 3] = {
    48,18,59, 50,21,67, 51,24,74, 52,27,81, 53,30,88, 54,33,95, 55,36,102, 56,39,109,
    57,42,115, 58,45,121, 59,47,128, 60,50,134, 61,53,139, 62,56,145, 63,59,151, 63,62,156,
    64,64,162, 65,67,167, 65,70,172, 66,73,177, 66,75,181, 67,78,186, 68,81,191, 68,84,195,
    68,86,199, 69,89,203, 69,92,207, 69,94,211, 70,97,214, 70,100,218, 70,102,221, 70,105,224,
    70,107,227, 71,110,230, 71,113,233, 71,115,235, 71,118,238, 71,120,240, 71,123,242, 70,125,244,
    70,128,246, 70,130,248, 70,133,250, 70,135,251, 69,138,252, 69,140,253, 68,143,254, 67,145,254,
    66,148,255, 65,150,255, 64,153,255, 62,155,254, 61,158,254, 59,160,253, 58,163,252, 56,165,251,
    55,168,250, 53,171,248, 51,173,247, 49,175,245, 47,178,244, 46,180,242, 44,183,240, 42,185,238,
    40,188,235, 39,190,233, 37,192,231, 35,195,228, 34,197,226, 32,199,223, 31,201,221, 30,203,218,
    28,205,216, 27,208,213, 26,210,210, 26,212,208, 25,213,205, 24,215,202, 24,217,200, 24,219,197,
    24,221,194, 24,222,192, 24,224,189, 25,226,187, 25,227,185, 26,228,182, 28,230,180, 29,231,178,
    31,233,175, 32,234,172, 34,235,170, 37,236,167, 39,238,164, 42,239,161, 44,240,158, 47,241,155,
    50,242,152, 53,243,148, 56,244,145, 60,245,142, 63,246,138, 67,247,135, 70,248,132, 74,248,128,
    78,249,125, 82,250,122, 85,250,118, 89,251,115, 93,252,111, 97,252,108, 101,253,105, 105,253,102,
    109,254,98, 113,254,95, 117,254,92, 121,254,89, 125,255,86, 128,255,83, 132,255,81, 136,255,78,
    139,255,75, 143,255,73, 146,255,71, 150,254,68, 153,254,66, 156,254,64, 159,253,63, 161,253,61,
    164,252,60, 167,252,58, 169,251,57, 172,251,56, 175,250,55, 177,249,54, 180,248,54, 183,247,53,
    185,246,53, 188,245,52, 190,244,52, 193,243,52, 195,241,52, 198,240,52, 200,239,52, 203,237,52,
    205,236,52, 208,234,52, 210,233,53, 212,231,53, 215,229,53, 217,228,54, 219,226,54, 221,224,55,
    223,223,55, 225,221,55, 227,219,56, 229,217,56, 231,215,57, 233,213,57, 235,211,57, 236,209,58,
    238,207,58, 239,205,58, 241,203,58, 242,201,58, 244,199,58, 245,197,58, 246,195,58, 247,193,58,
    248,190,57, 249,188,57, 250,186,57, 251,184,56, 251,182,55, 252,179,54, 252,177,54, 253,174,53,
    253,172,52, 254,169,51, 254,167,50, 254,164,49, 254,161,48, 254,158,47, 254,155,45, 254,153,44,
    254,150,43, 254,147,42, 254,144,41, 253,141,39, 253,138,38, 252,135,37, 252,132,35, 251,129,34,
    251,126,33, 250,123,31, 249,120,30, 249,117,29, 248,114,28, 247,111,26, 246,108,25, 245,105,24,
    244,102,23, 243,99,21, 242,96,20, 241,93,19, 240,91,18, 239,88,17, 237,85,16, 236,83,15,
    235,80,14, 234,78,13, 232,75,12, 231,73,12, 229,71,11, 228,69,10, 226,67,10, 225,65,9,
    223,63,8, 221,61,8, 220,59,7, 218,57,7, 216,55,6, 214,53,6, 212,51,5, 210,49,5,
    208,47,5, 206,45,4, 204,43,4, 202,42,4, 200,40,3, 197,38,3, 195,37,3, 193,35,2,
    190,33,2, 188,32,2, 185,30,2, 183,29,2, 180,27,1, 178,26,1, 175,24,1, 172,23,1,
    169,22,1, 167,20,1, 164,19,1, 161,18,1, 158,16,1, 155,15,1, 152,14,1, 149,13,1,
    146,11,1, 142,10,1, 139,9,2, 136,8,2, 133,7,2, 129,6,2, 126,5,2, 122,4,3,
};

__device__ __forceinline__ int gray(int r, int g, int b) { return (9798 * r + 19235 * g + 3735 * b + 16384) >> 15; }

__device__ __forceinline__ int div255(int t) {
  t += 128;
  return ((t >> 8) + t) >> 8;
}

// ------------------------------------------------------------------------------------------- heat-map colours
__global__ void __launch_bounds__(kThreads)
heat_kernel(const long long* __restrict__ off, const uint8_t* __restrict__ symmetric, const float* __restrict__ values,
            float max_distance, float* __restrict__ colors) {
  __shared__ unsigned red[2][kThreads / 32];
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long s0 = off[pair];
  const int n = (int)(off[pair + 1] - s0);                 // a slot is one object's vertices: < 2^31
  if (n <= 0) return;
  const bool sym = symmetric[pair] != 0;
  // every value is >= 0 or NaN (a distance), so the unsigned order of the bits is the float order with NaN on top
  unsigned lo = __float_as_uint(max_distance), hi = lo;
  if (sym) lo = 0u;
  for (int j = tid; j < n; j += kThreads) {
    const unsigned b = __float_as_uint(values[s0 + j]) & 0x7fffffffu;     // -0 -> +0
    lo = min(lo, b);
    hi = max(hi, b);
  }
  lo = __reduce_min_sync(0xffffffffu, lo);
  hi = __reduce_max_sync(0xffffffffu, hi);
  if (lane == 0) { red[0][warp] = lo; red[1][warp] = hi; }
  __syncthreads();
  lo = red[0][0];
  hi = red[1][0];
  for (int w = 1; w < kThreads / 32; ++w) { lo = min(lo, red[0][w]); hi = max(hi, red[1][w]); }
  const double md = (double)max_distance;
  const double dlo = __ddiv_rn((double)__uint_as_float(lo), md), dhi = __ddiv_rn((double)__uint_as_float(hi), md);
  const double range = __dsub_rn(dhi, dlo);
  const bool bad = hi > 0x7f800000u || !(range > 0.0);
  for (int j = tid; j < n; j += kThreads) {
    float* c = colors + 3 * (s0 + j);
    int k = -1;
    if (!bad) {
      const double d = __ddiv_rn((double)values[s0 + j], md);
      k = min((int)__dmul_rn(__ddiv_rn(__dsub_rn(d, dlo), range), 256.0), 255);   // x in [0, 1]: truncation floors
    }
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) c[ch] = k < 0 ? 0.f : __fdiv_rn((float)kTurbo[3 * k + ch], 255.f);
  }
}

// ------------------------------------------------------------------------------------------- overlay
struct LayerView {
  const float* alpha;
  int H, W;
  __device__ __forceinline__ bool in(int y, int x) const {
    return y >= 0 && y < H && x >= 0 && x < W && alpha[(size_t)y * W + x] > 0.f;
  }
  __device__ __forceinline__ bool edge(int y, int x) const {
    return in(y, x) && !(in(y - 1, x) && in(y + 1, x) && in(y, x - 1) && in(y, x + 1));
  }
};

__global__ void __launch_bounds__(kThreads)
overlay_kernel(int H, int W, int n_layers, const uint8_t* __restrict__ image, const float* __restrict__ renders,
               const long long* __restrict__ boxes, const uint8_t* __restrict__ colors, uint8_t* __restrict__ out) {
  const long long p = (long long)blockIdx.x * kThreads + threadIdx.x;
  const long long plane = (long long)H * W;
  if (p >= plane) return;
  const int y = (int)(p / W), x = (int)(p % W);
  int r = 0, g = 0, b = 0;
  if (image) r = g = b = gray(image[3 * p], image[3 * p + 1], image[3 * p + 2]);
  for (int l = 0; l < n_layers; ++l) {
    const long long* bx = boxes + 4 * (size_t)l;
    if (x < __ldg(bx) - 1 || y < __ldg(bx + 1) - 1 || x >= __ldg(bx + 2) || y >= __ldg(bx + 3)) continue;
    const float* rl = renders + (size_t)l * 4 * plane;
    const LayerView v{rl + 3 * plane, H, W};
    if (rl[3 * plane + p] > 0.f) {
      r = (int)rintf(__fmul_rn(rl[p], 255.f));
      g = (int)rintf(__fmul_rn(rl[plane + p], 255.f));
      b = (int)rintf(__fmul_rn(rl[2 * plane + p], 255.f));
    }
    if (colors && (v.edge(y, x) || v.edge(y, x + 1) || v.edge(y + 1, x) || v.edge(y + 1, x + 1))) {
      r = colors[3 * l];
      g = colors[3 * l + 1];
      b = colors[3 * l + 2];
    }
  }
  out[3 * p] = (uint8_t)min(max(r, 0), 255);
  out[3 * p + 1] = (uint8_t)min(max(g, 0), 255);
  out[3 * p + 2] = (uint8_t)min(max(b, 0), 255);
}

// ------------------------------------------------------------------------------------------- Kabsch panels
// np.uint8 of an fp32 value: truncation to int32 (cvttss2si: INT_MIN outside the range and for NaN), low 8 bits
__device__ __forceinline__ int np_uint8(float v) { return fabsf(v) < 2147483648.f ? __float2int_rz(v) & 255 : 0; }

// convert_tensor_to_image of channel c of a normalised crop
__device__ __forceinline__ int unnormalise(float v, int c) {
  const float mean = c == 0 ? (float)(-0.485 / 0.229) : c == 1 ? (float)(-0.456 / 0.224) : (float)(-0.406 / 0.225);
  const float std = c == 0 ? (float)(1 / 0.229) : c == 1 ? (float)(1 / 0.224) : (float)(1 / 0.225);
  return np_uint8(__fmul_rn(__fdiv_rn(__fsub_rn(v, mean), std), 255.f));
}

struct Warp {
  double m[6];                                            // the inverse map, cv2's iM
  __device__ void init(const float* M) {
    const double a = M[0], b = M[1], c = M[2], d = M[3], e = M[4], f = M[5];
    double D = __dsub_rn(__dmul_rn(a, e), __dmul_rn(b, d));
    D = D != 0.0 ? __ddiv_rn(1.0, D) : 0.0;
    const double A11 = __dmul_rn(e, D), A22 = __dmul_rn(a, D), A12 = __dmul_rn(b, -D), A21 = __dmul_rn(d, -D);
    m[0] = A11; m[1] = A12; m[3] = A21; m[4] = A22;
    m[2] = __dsub_rn(__dmul_rn(-A11, c), __dmul_rn(A12, f));
    m[5] = __dsub_rn(__dmul_rn(-A21, c), __dmul_rn(A22, f));
  }
  // source pixel (sx, sy) and fractions (fx, fy) in 1/32 of destination pixel (x, y)
  __device__ __forceinline__ void map(int x, int y, int& sx, int& sy, int& fx, int& fy) const {
    const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)y), m[2]), 1024.0)) + 16;
    const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)y), m[5]), 1024.0)) + 16;
    const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)x), 1024.0))) >> 5;
    const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)x), 1024.0))) >> 5;
    sx = min(max(X >> 5, -32768), 32767);
    sy = min(max(Y >> 5, -32768), 32767);
    fx = X & 31;
    fy = Y & 31;
  }
};

// bilinear tap sum of one u8 channel, produced by `get(y, x)` inside the crop (0 outside)
template <class F>
__device__ __forceinline__ int bilinear(int sx, int sy, int fx, int fy, F get) {
  const int w[4] = {32 * (32 - fx) * (32 - fy), 32 * fx * (32 - fy), 32 * (32 - fx) * fy, 32 * fx * fy};
  int s = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int yy = sy + (k >> 1), xx = sx + (k & 1);
    if (yy >= 0 && yy < kCrop && xx >= 0 && xx < kCrop) s += w[k] * get(yy, xx);
  }
  return min((s + 16384) >> 15, 255);
}

__global__ void __launch_bounds__(kTile * kTile)
kabsch_kernel(const float* __restrict__ query, const float* __restrict__ query_mask, const float* __restrict__ tmpl,
              const float* __restrict__ tmpl_mask, const float* __restrict__ Ms, uint8_t* __restrict__ out) {
  __shared__ uint8_t sWarp[kHalo][kHalo], sQuery[kHalo][kHalo];     // DIV255(a a) > 0 of the two masks
  __shared__ uint8_t sAlpha[kTile][kTile];
  const int i = blockIdx.z, tx = threadIdx.x, ty = threadIdx.y, tid = ty * kTile + tx;
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const size_t plane = (size_t)kCrop * kCrop;
  const float* tm = tmpl_mask + i * plane;
  Warp wp;
  wp.init(Ms + 9 * (size_t)i);
  const auto alpha_at = [&](int x, int y) {
    int sx, sy, fx, fy;
    wp.map(x, y, sx, sy, fx, fy);
    return bilinear(sx, sy, fx, fy, [&](int yy, int xx) { return np_uint8(__fmul_rn(tm[yy * kCrop + xx], 255.f)); });
  };
  for (int k = tid; k < kHalo * kHalo; k += kTile * kTile) {
    const int hy = k / kHalo, hx = k % kHalo, y = y0 + hy - 2, x = x0 + hx - 2;
    uint8_t w = 0, q = 0;
    if (y >= 0 && y < kCrop && x >= 0 && x < kCrop) {
      const int a = alpha_at(x, y);
      const int qm = np_uint8(__fmul_rn(query_mask[i * plane + (size_t)y * kCrop + x], 255.f));
      w = div255(a * a) > 0;
      q = div255(qm * qm) > 0;
      if (hy >= 2 && hy < kTile + 2 && hx >= 2 && hx < kTile + 2) sAlpha[hy - 2][hx - 2] = (uint8_t)a;
    }
    sWarp[hy][hx] = w;
    sQuery[hy][hx] = q;
  }
  __syncthreads();
  const int x = x0 + tx, y = y0 + ty;
  // halo (hy, hx) holds pixel (y0 + hy - 2, x0 + hx - 2); outside the crop it holds 0, which is "outside the mask"
  const auto edge3 = [&](uint8_t (*m)[kHalo]) {
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int hy = ty + 2 + dy, hx = tx + 2 + dx;
        if (m[hy][hx] && !(m[hy - 1][hx] && m[hy + 1][hx] && m[hy][hx - 1] && m[hy][hx + 1])) return true;
      }
    return false;
  };
  const size_t p = (size_t)y * kCrop + x;
  const float* q = query + i * 3 * plane;
  const int gq = gray(unnormalise(q[p], 0), unnormalise(q[plane + p], 1), unnormalise(q[2 * plane + p], 2));
  const int a = sAlpha[ty][tx];
  int sx, sy, fx, fy;
  wp.map(x, y, sx, sy, fx, fy);
  int rgb[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* tc = tmpl + (i * 3 + c) * plane;
    const int w = bilinear(sx, sy, fx, fy, [&](int yy, int xx) { return unnormalise(tc[yy * kCrop + xx], c); });
    rgb[c] = div255(gq * (255 - a) + w * a);
  }
  if (edge3(sWarp)) { rgb[0] = 255; rgb[1] = 0; rgb[2] = 0; }
  if (edge3(sQuery)) { rgb[0] = 0; rgb[1] = 255; rgb[2] = 0; }
  uint8_t* o = out + 3 * (i * plane + p);
  o[0] = (uint8_t)rgb[0];
  o[1] = (uint8_t)rgb[1];
  o[2] = (uint8_t)rgb[2];
}

}  // namespace

extern "C" int gp_vis_vertex_errors(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets,
                                    const float* vertices, const float* pose_est, const float* pose_gt,
                                    const uint8_t* symmetric, const int64_t* out_offsets, float* values, void* stream) {
  if (n_pairs < 1) return fail(GP_ERR_INVALID, "n_pairs %d must be >= 1", n_pairs);
  if (n_pairs > 65535 * 32768) return fail(GP_ERR_INVALID, "n_pairs %d too large", n_pairs);
  if (n_objects < 1 || n_objects > GP_BOP_MAX_OBJECTS)
    return fail(GP_ERR_INVALID, "n_objects %d outside [1, %d]", n_objects, GP_BOP_MAX_OBJECTS);
  if (!vertex_offsets) return fail(GP_ERR_INVALID, "null offsets");
  int max_v = 0;
  for (int o = 0; o <= n_objects; ++o) {
    if (o == 0 ? vertex_offsets[0] != 0 : vertex_offsets[o] <= vertex_offsets[o - 1])
      return fail(GP_ERR_INVALID, "bad vertex offsets at object %d: they must start at 0 and increase strictly", o);
    if (o > 0) max_v = max(max_v, vertex_offsets[o] - vertex_offsets[o - 1]);
  }
  if ((max_v + GP_BOP_ADD_CHUNK - 1) / GP_BOP_ADD_CHUNK > 65535)
    return fail(GP_ERR_INVALID, "an object of %d vertices has more than 65535 chunks", max_v);
  if (!obj_idx || !vertices || !pose_est || !pose_gt || !symmetric || !out_offsets || !values)
    return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_add_vertex_errors(n_pairs, n_objects, obj_idx, vertex_offsets, vertices, pose_est, pose_gt,
                                       symmetric, out_offsets, values, static_cast<cudaStream_t>(stream)));
  return GP_OK;
}

extern "C" int gp_vis_heat_colors(int n_pairs, const int64_t* offsets, const uint8_t* symmetric, const float* values,
                                  float max_distance, float* colors, void* stream) {
  if (n_pairs < 1) return fail(GP_ERR_INVALID, "n_pairs %d must be >= 1", n_pairs);
  if (!(max_distance > 0.f) || !isfinite(max_distance))
    return fail(GP_ERR_INVALID, "max_distance must be positive and finite");
  if (!offsets || !symmetric || !values || !colors) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(heat_kernel, n_pairs, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false,
                        reinterpret_cast<const long long*>(offsets), symmetric, values, max_distance, colors));
  return GP_OK;
}

extern "C" int gp_vis_overlay(int height, int width, int n_layers, const uint8_t* image, const float* renders,
                              const int64_t* boxes, const uint8_t* colors, uint8_t* out, void* stream) {
  if (height < 1 || width < 1 || height > GP_VIS_MAX_SIDE || width > GP_VIS_MAX_SIDE)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [1, %d]", height, width, GP_VIS_MAX_SIDE);
  if (n_layers < 0) return fail(GP_ERR_INVALID, "n_layers %d must be >= 0", n_layers);
  if (n_layers > 0 && (!renders || !boxes)) return fail(GP_ERR_INVALID, "null renders or boxes");
  if (!out) return fail(GP_ERR_INVALID, "null out");
  const long long n = (long long)height * width;
  GP_CUDA(gp::launch_ex(overlay_kernel, (unsigned)((n + kThreads - 1) / kThreads), kThreads, 0,
                        static_cast<cudaStream_t>(stream), 1, false, height, width, n_layers, image, renders,
                        reinterpret_cast<const long long*>(boxes), colors, out));
  return GP_OK;
}

extern "C" int gp_vis_kabsch(int n, const float* query, const float* query_mask, const float* tmpl,
                             const float* tmpl_mask, const float* M, uint8_t* out, void* stream) {
  if (n < 1 || n > 65535) return fail(GP_ERR_INVALID, "n %d outside [1, 65535]", n);
  if (!query || !query_mask || !tmpl || !tmpl_mask || !M || !out) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(kabsch_kernel, dim3(kCrop / kTile, kCrop / kTile, n), dim3(kTile, kTile), 0,
                        static_cast<cudaStream_t>(stream), 1, false, query, query_mask, tmpl, tmpl_mask, M, out));
  return GP_OK;
}
