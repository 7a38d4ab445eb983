// Row f5 of SURVEY.md §8: template renders from a CAD mesh on the GPU.  The reference renders the 162 templates of
// an object with Panda3D (src/custom_megapose/call_panda3d.py:45-59: 640 x 480, the fixed template intrinsics, one
// white ambient light, i.e. the image is the surface albedo; 4x multisampling, two-sided faces, black transparent
// background), writes PNGs and reads them back to take the mask (depth > 0) and the PIL bounding box
// (custom_megapose/template_dataset.py:66-119).  Here one call renders n views of one triangle mesh straight into the
// RGBA / depth / box tensors that gp_crop_resize_pad takes.
//
// Contract (what tests/test_gpu_render.py pins against oracle/render_port.py):
//  - Camera, OpenCV convention: p = R X + t with the object->camera pose [R|t] (row-major 4x4),
//    u = (K00 x + K01 y) / z + K02, v = K11 y / z + K12.  Pixel (i, j) = (column, row) is centred at (i, j); its 4
//    samples sit at the rotated-grid offsets (-1/8,-3/8), (3/8,-1/8), (-3/8,1/8), (1/8,3/8) from the centre.
//  - Coverage is exact and schedule-independent: u, v are computed in fp32, snapped to 1/256 px (round to nearest
//    even), and the edge functions are evaluated in 64-bit integers with the top-left fill rule.  Both windings are
//    rasterised (two-sided): a triangle is put in positive-area order, then rotated to start at its smallest snapped
//    (y, x), so every corner order of the same triangle gives the same arithmetic.  Zero-area triangles are skipped.
//    A triangle with any vertex at z <= z_near, with a vertex index outside [0, V), or with a vertex projected more
//    than 2^22 px from the origin (keeps every edge product inside int64) is dropped, not clipped.
//  - Visibility: per-sample depth z = 1 / sum_i (lambda_i / z_i), lambda_i = float(w_i) / float(2A) from the integer
//    edge values, in fp32 with the operation order written below and no FMA contraction.  It is resolved with a
//    64-bit atomicMin on (float bits of z) << 32 | face id: the nearest surface wins, on an exact depth tie the lowest
//    face id, whatever the launch order.  The key buffer alone decides the output, so it is bit-identical run to run.
//  - Shading, albedo only: per-vertex colour [V,3], or a texture [Ht,Wt,3] (row 0 = top) with per-face-corner UV
//    [F,3,2] sampled bilinearly at level 0 with repeat wrap and v = 0 at the bottom row, or a constant colour (white
//    when NULL).  Attributes are interpolated perspective-correctly: a = (sum_i lambda_i / z_i * a_i) * z.
//  - Resolve, one thread per pixel: RGB = round(255 * mean of the 4 samples (background = 0)) / 255, the 8-bit
//    framebuffer + PNG round trip; alpha = 1 if any sample is covered; depth = the smallest covered sample z, else 0.
//  - Boxes: [x0, y0, x1, y1) of alpha > 0 with exclusive max (PIL getbbox), (0, 0, W, H) for an empty view.
//  - Depth only (gp_render_depth, the depth maps of the BOP pose-error metrics): the same raster with ONE sample per
//    pixel at offset (0, 0), i.e. at the pixel centre as the BOP renderers take it; depth = that sample's z (0 =
//    background), boxes of depth > 0; no shading and no RGBA.  The sample count is a template parameter of the raster
//    and resolve code, so both entry points share every line of the arithmetic above.
//
// Layout: one thread per (view, face) sets the triangle up and rasterises it alone when its pixel bounding box is at
// most kSmallPixels; larger triangles are queued in shared memory and rasterised by the whole CTA, so neither a mesh
// of 10^6 sub-pixel faces nor one of a few screen-filling faces serialises on one thread.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kSmallPixels = 32;
constexpr float kGuardPx = 4194304.f;                    // 2^22 px: snapped |coordinate| < 2^30
constexpr unsigned long long kEmpty = ~0ull;

// sample offsets in 1/256 px: the rotated grid of 4x MSAA, or the pixel centre for one sample
template <int NS>
__device__ __forceinline__ int sample_dx(int s) { return NS == 1 ? 0 : s == 0 ? -32 : s == 1 ? 96 : s == 2 ? -96 : 32; }
template <int NS>
__device__ __forceinline__ int sample_dy(int s) { return NS == 1 ? 0 : s == 0 ? -96 : s == 1 ? -32 : s == 2 ? 32 : 96; }
// largest |offset| of a sample from its pixel centre, 1/256 px
template <int NS>
constexpr int sample_reach() { return NS == 1 ? 0 : 96; }

struct Tri {
  int x[3], y[3];          // snapped screen positions (1/256 px), ordered so that the doubled area is positive
  float iz[3];             // 1 / z
  int corner[3];           // face corner (0..2) of each slot
  long long area;          // doubled area, > 0
};

// a[k] <- a[(k + r) % 3] with constant indices only, so that the triangle stays in registers
template <class T>
__device__ __forceinline__ void rotate3(T (&a)[3], int r) {
  const T a0 = a[0], a1 = a[1], a2 = a[2];
  a[0] = r == 0 ? a0 : r == 1 ? a1 : a2;
  a[1] = r == 0 ? a1 : r == 1 ? a2 : a0;
  a[2] = r == 0 ? a2 : r == 1 ? a0 : a1;
}

// Projects the three corners of face f and orders them; false if the face is dropped.
__device__ __forceinline__ bool setup_triangle(int f, int nv, const float* __restrict__ V, const int* __restrict__ faces,
                                               const float* P, const float* K, float z_near, Tri& t) {
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const int vi = faces[3 * (size_t)f + k];
    if (vi < 0 || vi >= nv) return false;
    const float X = V[3 * (size_t)vi], Y = V[3 * (size_t)vi + 1], Z = V[3 * (size_t)vi + 2];
    const float x = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[0], X), __fmul_rn(P[1], Y)), __fmul_rn(P[2], Z)), P[3]);
    const float y = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[4], X), __fmul_rn(P[5], Y)), __fmul_rn(P[6], Z)), P[7]);
    const float z = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[8], X), __fmul_rn(P[9], Y)), __fmul_rn(P[10], Z)), P[11]);
    if (!(z > z_near)) return false;                                   // also drops NaN
    const float u = __fadd_rn(__fdiv_rn(__fadd_rn(__fmul_rn(K[0], x), __fmul_rn(K[1], y)), z), K[2]);
    const float v = __fadd_rn(__fdiv_rn(__fmul_rn(K[4], y), z), K[5]);
    if (!(fabsf(u) < kGuardPx && fabsf(v) < kGuardPx)) return false;
    t.x[k] = __float2int_rn(__fmul_rn(u, 256.f));
    t.y[k] = __float2int_rn(__fmul_rn(v, 256.f));
    t.iz[k] = __frcp_rn(z);
    t.corner[k] = k;
  }
  long long a = ((long long)t.x[1] - t.x[0]) * ((long long)t.y[2] - t.y[0]) -
                ((long long)t.y[1] - t.y[0]) * ((long long)t.x[2] - t.x[0]);
  if (a == 0) return false;
  if (a < 0) {                                                         // the other winding: swap slots 1 and 2
    int s = t.x[1]; t.x[1] = t.x[2]; t.x[2] = s;
    s = t.y[1]; t.y[1] = t.y[2]; t.y[2] = s;
    const float z = t.iz[1]; t.iz[1] = t.iz[2]; t.iz[2] = z;
    t.corner[1] = 2; t.corner[2] = 1;
    a = -a;
  }
  t.area = a;
  // start at the vertex with the smallest (y, x): the same triangle listed in any corner order or winding then sums
  // its depth terms in one order, so coplanar duplicates tie exactly and the face id decides
  int r = 0;
  if (t.y[1] < t.y[r] || (t.y[1] == t.y[r] && t.x[1] < t.x[r])) r = 1;
  if (t.y[2] < t.y[r] || (t.y[2] == t.y[r] && t.x[2] < t.x[r])) r = 2;
  rotate3(t.x, r); rotate3(t.y, r); rotate3(t.iz, r); rotate3(t.corner, r);
  return true;
}

// Edge function of a -> b at p; with the top-left rule a sample on the edge is inside iff the edge is a top edge
// (dy == 0, dx > 0: the interior lies below it) or a left edge (dy < 0).  Returns -1 for "outside".
__device__ __forceinline__ long long edge(int ax, int ay, int bx, int by, int px, int py) {
  const long long dx = (long long)bx - ax, dy = (long long)by - ay;
  const long long e = dx * ((long long)py - ay) - dy * ((long long)px - ax);
  const bool top_left = dy < 0 || (dy == 0 && dx > 0);
  return (e > 0 || (e == 0 && top_left)) ? e : -1;
}

// lambda_i / z_i of the sample at (sx, sy); false if the sample is outside
__device__ __forceinline__ bool sample_weights(const Tri& t, int sx, int sy, float b[3]) {
  const long long w0 = edge(t.x[1], t.y[1], t.x[2], t.y[2], sx, sy);
  const long long w1 = edge(t.x[2], t.y[2], t.x[0], t.y[0], sx, sy);
  const long long w2 = edge(t.x[0], t.y[0], t.x[1], t.y[1], sx, sy);
  if (w0 < 0 || w1 < 0 || w2 < 0) return false;
  const float a = __ll2float_rn(t.area);
  b[0] = __fmul_rn(__fdiv_rn(__ll2float_rn(w0), a), t.iz[0]);
  b[1] = __fmul_rn(__fdiv_rn(__ll2float_rn(w1), a), t.iz[1]);
  b[2] = __fmul_rn(__fdiv_rn(__ll2float_rn(w2), a), t.iz[2]);
  return true;
}

__device__ __forceinline__ float sample_depth(const float b[3]) {
  return __frcp_rn(__fadd_rn(__fadd_rn(b[0], b[1]), b[2]));
}

template <int NS>
__device__ __forceinline__ void raster_pixel(const Tri& t, int face, int px, int py, int W,
                                             unsigned long long* __restrict__ keys) {
  unsigned long long* k = keys + ((size_t)py * W + px) * NS;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    float b[3];
    if (!sample_weights(t, px * 256 + sample_dx<NS>(s), py * 256 + sample_dy<NS>(s), b)) continue;
    const unsigned long long key =
        ((unsigned long long)__float_as_uint(sample_depth(b)) << 32) | (unsigned long long)(unsigned)face;
    atomicMin(k + s, key);
  }
}

__device__ __forceinline__ int floor_div256(int a) { return a >> 8; }   // arithmetic shift == floor division

template <int NS>
__global__ void __launch_bounds__(kThreads)
raster_kernel(int H, int W, int nv, const float* __restrict__ V, int nf, const int* __restrict__ faces,
              const float* __restrict__ poses, const float* __restrict__ Kmat, float z_near,
              unsigned long long* __restrict__ keys) {
  __shared__ float sP[12], sK[6];
  __shared__ Tri big[kThreads];
  __shared__ int big_face[kThreads], big_box[kThreads][4];
  __shared__ int nbig;
  const int view = blockIdx.y, tid = threadIdx.x;
  if (tid < 12) sP[tid] = poses[16 * (size_t)view + tid];
  if (tid < 6) sK[tid] = Kmat[tid];
  if (tid == 0) nbig = 0;
  __syncthreads();
  keys += (size_t)view * H * W * NS;
  const int f = blockIdx.x * kThreads + tid;
  Tri t;
  if (f < nf && setup_triangle(f, nv, V, faces, sP, sK, z_near, t)) {
    const int xmin = min(min(t.x[0], t.x[1]), t.x[2]), xmax = max(max(t.x[0], t.x[1]), t.x[2]);
    const int ymin = min(min(t.y[0], t.y[1]), t.y[2]), ymax = max(max(t.y[0], t.y[1]), t.y[2]);
    // pixel i holds samples at 256 i + [-reach, reach]
    constexpr int R = sample_reach<NS>();
    const int px0 = max(-floor_div256(R - xmin), 0), px1 = min(floor_div256(xmax + R), W - 1);
    const int py0 = max(-floor_div256(R - ymin), 0), py1 = min(floor_div256(ymax + R), H - 1);
    if (px0 <= px1 && py0 <= py1) {
      if ((long long)(px1 - px0 + 1) * (py1 - py0 + 1) <= kSmallPixels) {
        for (int py = py0; py <= py1; ++py)
          for (int px = px0; px <= px1; ++px) raster_pixel<NS>(t, f, px, py, W, keys);
      } else {
        const int slot = atomicAdd(&nbig, 1);                // queue order is irrelevant: atomicMin decides
        big[slot] = t;
        big_face[slot] = f;
        big_box[slot][0] = px0; big_box[slot][1] = py0; big_box[slot][2] = px1 - px0 + 1; big_box[slot][3] = py1 - py0 + 1;
      }
    }
  }
  __syncthreads();
  for (int i = 0; i < nbig; ++i) {
    const int bw = big_box[i][2], n = bw * big_box[i][3];
    for (int p = tid; p < n; p += kThreads) {
      const int py = p / bw;
      raster_pixel<NS>(big[i], big_face[i], big_box[i][0] + p - py * bw, big_box[i][1] + py, W, keys);
    }
  }
}

__device__ __forceinline__ float lerp_rn(float a, float b, float w) {
  return __fadd_rn(__fmul_rn(__fsub_rn(1.f, w), a), __fmul_rn(w, b));
}

// wraps an integral float into [0, n)
__device__ __forceinline__ int wrap_index(float i, int n) {
  float m = fmodf(i, (float)n);                                        // exact
  if (m < 0.f) m = __fadd_rn(m, (float)n);
  const int r = (int)m;
  return r >= n ? 0 : r;
}

// bilinear, level 0, repeat; texel (c, r) of a [th, tw] texture with row 0 on top has its centre at
// u = (c + 0.5) / tw, v = (th - 1 - r + 0.5) / th
__device__ void sample_texture(const float* __restrict__ tex, int th, int tw, float u, float v, float rgb[3]) {
  float fx = __fsub_rn(__fmul_rn(u, (float)tw), 0.5f);
  float fy = __fsub_rn(__fmul_rn(v, (float)th), 0.5f);
  if (!isfinite(fx)) fx = 0.f;
  if (!isfinite(fy)) fy = 0.f;
  const float x0 = floorf(fx), y0 = floorf(fy);
  const float ax = __fsub_rn(fx, x0), ay = __fsub_rn(fy, y0);
  const int c0 = wrap_index(x0, tw), c1 = c0 + 1 == tw ? 0 : c0 + 1;
  const int b0 = wrap_index(y0, th), b1 = b0 + 1 == th ? 0 : b0 + 1;      // rows counted from the bottom
  const float* r0 = tex + (size_t)(th - 1 - b0) * tw * 3;
  const float* r1 = tex + (size_t)(th - 1 - b1) * tw * 3;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float lo = lerp_rn(r0[3 * c0 + c], r0[3 * c1 + c], ax);
    const float hi = lerp_rn(r1[3 * c0 + c], r1[3 * c1 + c], ax);
    rgb[c] = lerp_rn(lo, hi, ay);
  }
}

__device__ __forceinline__ float interpolate(const float b[3], float z, float a0, float a1, float a2) {
  return __fmul_rn(__fadd_rn(__fadd_rn(__fmul_rn(b[0], a0), __fmul_rn(b[1], a1)), __fmul_rn(b[2], a2)), z);
}

// kShade = false: depth only (rgba and the shading inputs are not read)
template <int NS, bool kShade>
__global__ void __launch_bounds__(kThreads)
resolve_kernel(int H, int W, int nv, const float* __restrict__ V, const int* __restrict__ faces,
               const float* __restrict__ vcolor, const float* __restrict__ face_uv, const float* __restrict__ tex,
               int th, int tw, const float* __restrict__ ccolor, const float* __restrict__ poses,
               const float* __restrict__ Kmat, float z_near, const unsigned long long* __restrict__ keys,
               float* __restrict__ rgba, float* __restrict__ depth) {
  __shared__ float sP[12], sK[6], sC[3];
  const int view = blockIdx.y, tid = threadIdx.x;
  if (tid < 12) sP[tid] = poses[16 * (size_t)view + tid];
  if (tid < 6) sK[tid] = Kmat[tid];
  if (tid < 3) sC[tid] = ccolor ? ccolor[tid] : 1.f;
  __syncthreads();
  const int pix = blockIdx.x * kThreads + tid;
  if (pix >= H * W) return;
  const int py = pix / W, px = pix - py * W;
  const unsigned long long* k = keys + ((size_t)view * H * W + pix) * NS;
  float sum[3] = {0.f, 0.f, 0.f};
  float zmin = 0.f;
  bool covered = false;
  for (int s = 0; s < NS; ++s) {
    const unsigned long long key = k[s];
    if (key == kEmpty) continue;                                       // background sample: adds 0
    const int f = (int)(unsigned)(key & 0xffffffffull);
    const float zs = __uint_as_float((unsigned)(key >> 32));
    zmin = covered ? fminf(zmin, zs) : zs;
    covered = true;
    if (!kShade) continue;
    Tri t;
    float b[3], c[3];
    setup_triangle(f, nv, V, faces, sP, sK, z_near, t);               // same arithmetic as the raster pass
    sample_weights(t, px * 256 + sample_dx<NS>(s), py * 256 + sample_dy<NS>(s), b);
    const float z = sample_depth(b);
    if (tex) {
      const float* uv = face_uv + 6 * (size_t)f;
      const float u = interpolate(b, z, uv[2 * t.corner[0]], uv[2 * t.corner[1]], uv[2 * t.corner[2]]);
      const float v = interpolate(b, z, uv[2 * t.corner[0] + 1], uv[2 * t.corner[1] + 1], uv[2 * t.corner[2] + 1]);
      sample_texture(tex, th, tw, u, v, c);
    } else if (vcolor) {
      const int* fv = faces + 3 * (size_t)f;
      const float* c0 = vcolor + 3 * (size_t)fv[t.corner[0]];
      const float* c1 = vcolor + 3 * (size_t)fv[t.corner[1]];
      const float* c2 = vcolor + 3 * (size_t)fv[t.corner[2]];
      for (int ch = 0; ch < 3; ++ch) c[ch] = interpolate(b, z, c0[ch], c1[ch], c2[ch]);
    } else {
      c[0] = sC[0]; c[1] = sC[1]; c[2] = sC[2];
    }
    for (int ch = 0; ch < 3; ++ch) sum[ch] = __fadd_rn(sum[ch], c[ch]);
  }
  const size_t plane = (size_t)H * W;
  if (kShade) {
    static_assert(!kShade || NS == 4, "the shaded resolve averages 4 samples");
    float* out = rgba + (size_t)view * 4 * plane + pix;
    for (int ch = 0; ch < 3; ++ch) {
      const float q = fminf(fmaxf(rintf(__fmul_rn(__fmul_rn(sum[ch], 0.25f), 255.f)), 0.f), 255.f);
      out[ch * plane] = __fdiv_rn(q, 255.f);
    }
    out[3 * plane] = covered ? 1.f : 0.f;
  }
  if (depth) depth[(size_t)view * plane + pix] = covered ? zmin : 0.f;
}

// one CTA per view: [x0, y0, x1, y1) of the pixels > 0 of the plane at mask + view * view_stride (alpha, or depth)
__global__ void __launch_bounds__(kThreads)
boxes_kernel(int H, int W, const float* __restrict__ mask, size_t view_stride, long long* __restrict__ boxes) {
  __shared__ int b[4];
  const int view = blockIdx.x;
  if (threadIdx.x == 0) { b[0] = W; b[1] = H; b[2] = -1; b[3] = -1; }
  __syncthreads();
  const float* alpha = mask + view * view_stride;
  int x0 = W, y0 = H, x1 = -1, y1 = -1;
  for (int p = threadIdx.x; p < H * W; p += kThreads) {
    if (alpha[p] > 0.f) {
      const int y = p / W, x = p - y * W;
      x0 = min(x0, x); x1 = max(x1, x); y0 = min(y0, y); y1 = max(y1, y);
    }
  }
  if (x1 >= 0) { atomicMin(&b[0], x0); atomicMin(&b[1], y0); atomicMax(&b[2], x1); atomicMax(&b[3], y1); }
  __syncthreads();
  if (threadIdx.x == 0) {
    long long* o = boxes + 4 * (size_t)view;
    const bool empty = b[2] < 0;
    o[0] = empty ? 0 : b[0]; o[1] = empty ? 0 : b[1];
    o[2] = empty ? W : b[2] + 1; o[3] = empty ? H : b[3] + 1;
  }
}

constexpr int kMaxSide = 8192;

int check_sizes(int max_views, int height, int width) {
  if (max_views < 0 || max_views > 65535) return fail(GP_ERR_INVALID, "n_views %d outside [0, 65535]", max_views);
  if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [1, %d]", height, width, kMaxSide);
  return GP_OK;
}

}  // namespace

extern "C" int gp_render_query_sizes(int max_views, int height, int width, size_t* workspace_bytes) {
  if (const int rc = check_sizes(max_views, height, width)) return rc;
  if (!workspace_bytes) return fail(GP_ERR_INVALID, "null workspace_bytes");
  *workspace_bytes = (size_t)max_views * height * width * 4 * sizeof(unsigned long long);
  return GP_OK;
}

extern "C" int gp_render_templates(int n_views, int height, int width, int num_vertices, const float* vertices,
                                   int num_faces, const int32_t* faces, const float* vertex_color, const float* face_uv,
                                   const float* texture, int tex_h, int tex_w, const float* constant_color,
                                   const float* poses, const float* K, float z_near, void* workspace, float* rgba,
                                   float* depth, int64_t* boxes, void* stream) {
  if (const int rc = check_sizes(n_views, height, width)) return rc;
  if (num_vertices < 0 || num_faces < 0) return fail(GP_ERR_INVALID, "negative mesh size");
  if (!(z_near > 0.f) || !isfinite(z_near)) return fail(GP_ERR_INVALID, "z_near must be positive and finite");
  if (!poses || !K || !workspace || !rgba || !boxes) return fail(GP_ERR_INVALID, "null argument");
  if (num_faces > 0 && (!vertices || !faces || num_vertices < 1))
    return fail(GP_ERR_INVALID, "null argument (mesh)");
  if (texture && vertex_color) return fail(GP_ERR_INVALID, "give vertex_color or texture, not both");
  if (texture && (!face_uv || tex_h < 1 || tex_w < 1))
    return fail(GP_ERR_INVALID, "texture needs face_uv and a positive tex_h x tex_w");
  if (face_uv && !texture) return fail(GP_ERR_INVALID, "face_uv without texture");
  if (n_views == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto* keys = static_cast<unsigned long long*>(workspace);
  const size_t key_bytes = (size_t)n_views * height * width * 4 * sizeof(unsigned long long);
  GP_CUDA(cudaMemsetAsync(keys, 0xFF, key_bytes, st));
  if (num_faces > 0)
    GP_CUDA(gp::launch_ex(raster_kernel<4>, dim3((num_faces + kThreads - 1) / kThreads, n_views), kThreads, 0, st, 1, false,
                          height, width, num_vertices, vertices, num_faces, faces, poses, K, z_near, keys));
  GP_CUDA(gp::launch_ex(resolve_kernel<4, true>, dim3((height * width + kThreads - 1) / kThreads, n_views), kThreads, 0, st, 1, false,
                        height, width, num_vertices, vertices, faces, vertex_color, face_uv, texture, tex_h, tex_w,
                        constant_color, poses, K, z_near, keys, rgba, depth));
  GP_CUDA(gp::launch_ex(boxes_kernel, n_views, kThreads, 0, st, 1, false, height, width, rgba + 3 * (size_t)height * width,
                        (size_t)4 * height * width, reinterpret_cast<long long*>(boxes)));
  return GP_OK;
}

extern "C" int gp_render_depth(int n_views, int height, int width, int num_vertices, const float* vertices,
                               int num_faces, const int32_t* faces, const float* poses, const float* K, float z_near,
                               void* workspace, float* depth, int64_t* boxes, void* stream) {
  if (const int rc = check_sizes(n_views, height, width)) return rc;
  if (num_vertices < 0 || num_faces < 0) return fail(GP_ERR_INVALID, "negative mesh size");
  if (!(z_near > 0.f) || !isfinite(z_near)) return fail(GP_ERR_INVALID, "z_near must be positive and finite");
  if (!poses || !K || !workspace || !depth || !boxes) return fail(GP_ERR_INVALID, "null argument");
  if (num_faces > 0 && (!vertices || !faces || num_vertices < 1))
    return fail(GP_ERR_INVALID, "null argument (mesh)");
  if (n_views == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto* keys = static_cast<unsigned long long*>(workspace);
  GP_CUDA(cudaMemsetAsync(keys, 0xFF, (size_t)n_views * height * width * sizeof(unsigned long long), st));
  if (num_faces > 0)
    GP_CUDA(gp::launch_ex(raster_kernel<1>, dim3((num_faces + kThreads - 1) / kThreads, n_views), kThreads, 0, st, 1, false,
                          height, width, num_vertices, vertices, num_faces, faces, poses, K, z_near, keys));
  GP_CUDA(gp::launch_ex(resolve_kernel<1, false>, dim3((height * width + kThreads - 1) / kThreads, n_views), kThreads, 0, st,
                        1, false, height, width, num_vertices, vertices, faces, nullptr, nullptr, nullptr, 0, 0, nullptr,
                        poses, K, z_near, keys, nullptr, depth));
  GP_CUDA(gp::launch_ex(boxes_kernel, n_views, kThreads, 0, st, 1, false, height, width, depth, (size_t)height * width,
                        reinterpret_cast<long long*>(boxes)));
  return GP_OK;
}
