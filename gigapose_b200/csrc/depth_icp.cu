// Row f6: depth refinement of the coarse poses, a GPU restatement of MegaPose's ICPRefiner
// (src/megapose/inference/icp_refiner.py:134-287, the `megapose-1.0-RGB-multi-hypothesis-icp` depth refiner).  One
// hypothesis is a (detection, pose) pair with: the measured depth D [H,W] of its frame (the unit of the pose
// translations, mm for BOP; 0 = missing), the frame's full-image K, an optional full-frame detection mask, the coarse
// pose T0 and the depth R [H,W] of the object rendered at T0 with that K (gp_render_templates, z_near = 0.1 m).  The
// reference's constants are in metres and are scaled by `unit_per_m`.
//
// Contract (what tests/test_gpu_icp.py pins against oracle/icp_port.py):
//  1. Scene, once per frame (gp_icp_prepare_scene).  S = Gaussian smoothing of D, sigma 2 px, radius 8 (scipy's
//     gaussian_filter, truncate 4), scipy's `reflect` border, as a normalised convolution: pixels with D <= 0 get
//     weight 0 and the weights are renormalised, S = (G * (D [D > 0])) / (G * [D > 0]) (0 where the denominator is 0),
//     vertical pass first.  Gradients g_v, g_u = np.gradient(S, 2, edge_order=2).  Normals are get_normal's
//     (icp_refiner.py:37-101): with a = u - cx, b = v - cy (not truncated), ix = 1/fx, iy = 1/fy,
//       t_u = (S ix + a ix g_u, b iy g_u, g_u),  t_v = (a ix g_v, S iy + b iy g_v, g_v),  n = cross(t_u, t_v) / |.|
//     (0 for a zero norm).  Points are back-projected from the raw D, x = ((u - cx) D) / fx, y = ((v - cy) D) / fy,
//     z = D, and the map stores z = 0 where D is outside (0.2 m, 5 m).  Target map f32 [F,H,W,6] = (x, y, z, n).
//  2. Target set: map z > 0 and the mask (icp_refiner.py:158-159); without a mask the reference's "threshold" rule
//     (refiner_utils.py:42-55): R > 0 and |D - R| <= 0.1 m.  Targets are counted over the whole frame with a mask and
//     over the render box without one (the rule needs R > 0).
//  3. Sources: targets with R > 0 (icp_refiner.py:176), back-projected from R like the targets, compacted in row-major
//     pixel order inside the render box.
//  4. Fewer than min_points targets or sources: status TOO_FEW_POINTS.  Otherwise t += mean(targets) - mean(sources)
//     (fp64 sums) and the source points move with it (icp_refiner.py:184-188).
//  5. ICP, levels L-1 .. 0 (L = 4), at most max_iters iterations each; level l uses every 2^l-th source in compacted
//     order.  Per iteration, with the current correction dT (fp64; its fp32 copy Tf transforms the sources):
//       association: s' = Tf s (fp32, ((T0 x + T1 y) + T2 z) + T3), u' = (fx x') / z' + cx, v' likewise, rounded to
//       nearest-even; the nearest valid target in 3-D (d2 = (dx dx + dy dy) + dz dz, fp32) in the (2 r_l + 1)^2 window,
//       r_l = 2^(l+1) px, clipped to the image; on a tie the lowest row-major index.  No target, or z' <= 0: no pair.
//       rejection: d = sqrt(d2); pairs with d > rejection_scale * median are dropped, median = the element of rank
//       (m - 1) / 2 of the m pair distances (exact, radix select on the float bits).
//       step: point-to-plane, linearised (Low 2004): r = (s' - q) . n, a = ((s' x n) / L, n) with L = 1 m, in fp64;
//       the 6x6 normal equations (sum a a^T) xi = -(sum a r) are accumulated per thread in index order, then by a
//       fixed shuffle tree and the warps in order, and solved by Cholesky; a pivot <= 1e-8 x the largest diagonal
//       entry ends the refinement with status DEGENERATE (a singular system: the surface does not constrain all six
//       degrees of freedom); no pair at all, or fewer than 6 kept pairs, with status LOST (the sources left the
//       target set: the pose diverged or started too far off).
//       update: omega = xi[0:3] / L, v = xi[3:6], dT <- [Rodrigues(omega) | v] dT; the level stops after a step with
//       |omega| < min_step_rad and |v| < min_step_m * unit_per_m.
//  6. residual = sqrt(sum r^2 / kept) of the last level-0 iteration, fitness = kept / level-0 sources.  The pose dT T0
//     (fp64, stored fp32) is written when residual <= max_residual * unit_per_m (status OK); otherwise, and on every
//     other status, out_pose is T0 bit for bit (icp_refiner.py:198-199, 283-284).
//
// Layout: three scene kernels (vertical pass, horizontal pass, normals) over all frames; one persistent CTA per
// hypothesis runs stages 2-6 without host synchronisation.  A hypothesis' result depends on its own inputs only.
//
// Masked normals (row f11, opt-in; the reference smooths the whole frame).  Detection d has a frame f, the measured
// depth D of f and a mask M_d, given dense or as COCO run-length encoding.
//  1'. Smoothing within the mask: S_d = (G * (D [D > 0] M_d)) / (G * ([D > 0] M_d)), the same G, vertical pass first,
//      scipy's `reflect` at the frame border, and the fp32 operation order of smooth_v_kernel / smooth_u_kernel.
//      Gradients and normals are stage 1's, taken from S_d; points are back-projected from the raw D as in stage 1.
//  2'. Target set: map z > 0 and M_d (stage 2's mask rule), counted over the mask's box.
//  Stages 3-6 are unchanged; hypothesis i reads the map and mask of detection det_idx[i], so the hypotheses of a
//  detection share them.
//  Consequences: with M_d = 1 over the frame the map is stage 1's bit for bit (skipping a weight-0 pixel adds +0).
//  Outside M_d every weight is 0, so S_d anywhere depends only on D inside the mask's bounding box [x0, x1) x [y0, y1),
//  and the map at the box's pixels only on S_d within 2 px of the box (the gradient stencil, one-sided at the frame
//  border).  So S_d is computed on the box grown by kMargin = 2 px and clipped to the frame ("ext"), the map and the
//  mask on the box itself, with box-relative addressing: memory scales with the box areas, not with H * W per
//  detection.  Layout: gp_icp_masked_decode writes the detection table and decodes each mask into a u8 box tile
//  (run-length masks: rle_scan_kernel's running sums, then the parity of the upper bound at col * H + row);
//  gp_icp_prepare_masked_scene runs three kernels over the ext tiles and boxes of all detections;
//  gp_icp_refine_masked is icp_kernel<true>, whose targets are looked up in the box tiles and whose scratch is
//  box-sized.  A pixel outside the box reads as 0 even where a dense mask is set: the box must contain the mask.
//
// Debug hooks (tests/test_gpu_icp_solver.py): with debug.trace set, thread 0 writes one gp_icp_trace_t per iteration
// (the fp32 transform it associated with, the counts, the median, the 29 fp64 sums, the step and the correction after
// it), so that each step can be checked against an fp64 reference started from the kernel's own state; the outputs are
// the same with and without it.  gp_debug_icp_select runs the median's radix_select alone.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

#include <algorithm>
#include <vector>

using gp::fail;

namespace {

constexpr int kScene = 256;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kRadius = 8;
constexpr int kAcc = 29;                 // 21 upper-triangle entries of A^T A, 6 of A^T r, sum r^2, kept pairs
constexpr int kMaxLevels = 8;
constexpr int kMinSide = 2 * kRadius + 1;
constexpr int kMaxSide = 8192;
constexpr unsigned kNoPair = 0x7f800000u;  // +inf bits: sorts after every distance
constexpr int kMargin = 2;               // ext = mask box + kMargin px: the gradient stencil, one-sided at the border

struct MaskDet {          // one detection of the masked mode (device table at the start of the masked workspace)
  int box[4];             // mask box x0, y0, x1, y1 (exclusive max); empty when x1 <= x0 or y1 <= y0
  int ext[4];             // the box grown by kMargin and clipped to the frame (empty with the box)
  int frame;
  int reserved;
  long long tile;         // first entry of its mask tile (u8) and map (f32 x 6), box-relative row-major
  long long ext_off;      // first entry of its num / den / S tiles, ext-relative row-major
  long long run0, run1;   // its runs in counts / ends (run-length masks)
};

__device__ __forceinline__ int reflect(int i, int n) {   // scipy 'reflect' (d c b a | a b c d | d c b a), n > kRadius
  return i < 0 ? -i - 1 : i >= n ? 2 * n - i - 1 : i;
}

// normalised Gaussian weights of scipy's _gaussian_kernel1d(2, 0, 8), rounded once to fp32
__device__ __forceinline__ void gauss_weights(float* w) {
  double e[2 * kRadius + 1], s = 0.0;
  for (int k = -kRadius; k <= kRadius; ++k) { e[k + kRadius] = exp(-0.5 * k * k / 4.0); s += e[k + kRadius]; }
  for (int k = 0; k <= 2 * kRadius; ++k) w[k] = (float)(e[k] / s);
}

// pass 1, along v: num = sum w D [D > 0], den = sum w [D > 0]
__global__ void __launch_bounds__(kScene)
smooth_v_kernel(int H, int W, const float* __restrict__ depth, float* __restrict__ num, float* __restrict__ den) {
  __shared__ float w[2 * kRadius + 1];
  if (threadIdx.x == 0) gauss_weights(w);
  __syncthreads();
  const size_t plane = (size_t)H * W;
  const int pix = blockIdx.x * kScene + threadIdx.x, f = blockIdx.y;
  if (pix >= H * W) return;
  const int v = pix / W, u = pix - v * W;
  const float* d = depth + f * plane;
  float sn = 0.f, sd = 0.f;
  for (int k = -kRadius; k <= kRadius; ++k) {
    const float z = d[(size_t)reflect(v + k, H) * W + u];
    if (z > 0.f) { sn = __fadd_rn(sn, __fmul_rn(w[k + kRadius], z)); sd = __fadd_rn(sd, w[k + kRadius]); }
  }
  num[f * plane + pix] = sn;
  den[f * plane + pix] = sd;
}

// pass 2, along u: S = (G_u * num) / (G_u * den)
__global__ void __launch_bounds__(kScene)
smooth_u_kernel(int H, int W, const float* __restrict__ num, const float* __restrict__ den, float* __restrict__ S) {
  __shared__ float w[2 * kRadius + 1];
  if (threadIdx.x == 0) gauss_weights(w);
  __syncthreads();
  const size_t plane = (size_t)H * W;
  const int pix = blockIdx.x * kScene + threadIdx.x, f = blockIdx.y;
  if (pix >= H * W) return;
  const int v = pix / W, u = pix - v * W;
  const float* a = num + f * plane + (size_t)v * W;
  const float* b = den + f * plane + (size_t)v * W;
  float sn = 0.f, sd = 0.f;
  for (int k = -kRadius; k <= kRadius; ++k) {
    const int j = reflect(u + k, W);
    sn = __fadd_rn(sn, __fmul_rn(w[k + kRadius], a[j]));
    sd = __fadd_rn(sd, __fmul_rn(w[k + kRadius], b[j]));
  }
  S[f * plane + pix] = sd > 0.f ? __fdiv_rn(sn, sd) : 0.f;
}

// np.gradient(x, 2, edge_order=2) at index i of a line of n samples with stride st
// x holds the samples lo, lo + 1, ... of the line (lo = 0: the whole line); every index read must be >= lo
__device__ __forceinline__ float gradient2(const float* x, int i, int n, int st, int lo = 0) {
  auto at = [&](int j) { return x[(size_t)(j - lo) * st]; };
  if (i == 0)
    return __fadd_rn(__fadd_rn(__fmul_rn(-0.75f, at(0)), at(1)), __fmul_rn(-0.25f, at(2)));
  if (i == n - 1)
    return __fadd_rn(__fadd_rn(__fmul_rn(0.25f, at(n - 3)), -at(n - 2)), __fmul_rn(0.75f, at(n - 1)));
  return __fdiv_rn(__fsub_rn(at(i + 1), at(i - 1)), 4.f);
}

// stage 1's map entry m[0..6) of pixel (u, v): smoothed depth z and its gradients gu, gv; raw depth d
__device__ __forceinline__ void map_entry(int u, int v, const float* K, float z, float gu, float gv, float d, float lo,
                                          float hi, float* m) {
  const float fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  const float a = __fsub_rn((float)u, cx), b = __fsub_rn((float)v, cy);
  const float ix = __frcp_rn(fx), iy = __frcp_rn(fy);
  const float tux = __fadd_rn(__fmul_rn(z, ix), __fmul_rn(__fmul_rn(a, ix), gu));
  const float tuy = __fmul_rn(__fmul_rn(b, iy), gu), tuz = gu;
  const float tvx = __fmul_rn(__fmul_rn(a, ix), gv);
  const float tvy = __fadd_rn(__fmul_rn(z, iy), __fmul_rn(__fmul_rn(b, iy), gv)), tvz = gv;
  float nx = __fsub_rn(__fmul_rn(tuy, tvz), __fmul_rn(tuz, tvy));
  float ny = __fsub_rn(__fmul_rn(tuz, tvx), __fmul_rn(tux, tvz));
  float nz = __fsub_rn(__fmul_rn(tux, tvy), __fmul_rn(tuy, tvx));
  const float nn = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(nx, nx), __fmul_rn(ny, ny)), __fmul_rn(nz, nz)));
  if (nn > 0.f) { nx = __fdiv_rn(nx, nn); ny = __fdiv_rn(ny, nn); nz = __fdiv_rn(nz, nn); }
  else { nx = ny = nz = 0.f; }
  const bool ok = d > lo && d < hi;
  m[0] = ok ? __fdiv_rn(__fmul_rn(a, d), fx) : 0.f;
  m[1] = ok ? __fdiv_rn(__fmul_rn(b, d), fy) : 0.f;
  m[2] = ok ? d : 0.f;
  m[3] = nx; m[4] = ny; m[5] = nz;
}

__global__ void __launch_bounds__(kScene)
normals_kernel(int H, int W, const float* __restrict__ depth, const float* __restrict__ Kmat, float lo, float hi,
               const float* __restrict__ S, float* __restrict__ map) {
  const size_t plane = (size_t)H * W;
  const int pix = blockIdx.x * kScene + threadIdx.x, f = blockIdx.y;
  if (pix >= H * W) return;
  const int v = pix / W, u = pix - v * W;
  const float* s = S + f * plane;
  const float gv = gradient2(s + u, v, H, W), gu = gradient2(s + (size_t)v * W, u, W, 1);
  map_entry(u, v, Kmat + 9 * f, s[pix], gu, gv, depth[f * plane + pix], lo, hi, map + (f * plane + pix) * 6);
}

// ---- masked normals (1'): one grid row per detection, box- or ext-relative pixel t of a tile
__device__ __forceinline__ bool in_box(const int* b, int u, int v) { return u >= b[0] && u < b[2] && v >= b[1] && v < b[3]; }

__global__ void __launch_bounds__(kScene)
mask_tiles_kernel(int H, int W, const MaskDet* __restrict__ dets, const uint8_t* __restrict__ dense,
                  const long long* __restrict__ ends, uint8_t* __restrict__ tiles) {
  const MaskDet& dt = dets[blockIdx.y];
  const int bw = dt.box[2] - dt.box[0], bh = dt.box[3] - dt.box[1];
  const int t = blockIdx.x * kScene + threadIdx.x;
  if (bw <= 0 || bh <= 0 || t >= bw * bh) return;
  const int v = dt.box[1] + t / bw, u = dt.box[0] + t % bw;
  const bool m = dense ? dense[(size_t)blockIdx.y * H * W + (size_t)v * W + u] != 0
                       : gp::rle_bit(ends, dt.run0, dt.run1, (long long)u * H + v);          // column-major runs
  tiles[dt.tile + t] = m;
}

// pass 1, along v, over the ext tile: num = sum w D [D > 0] M, den = sum w [D > 0] M (M = 0 outside the box)
__global__ void __launch_bounds__(kScene)
masked_smooth_v_kernel(int H, int W, const MaskDet* __restrict__ dets, const float* __restrict__ depth,
                       const uint8_t* __restrict__ tiles, float* __restrict__ num, float* __restrict__ den) {
  __shared__ float w[2 * kRadius + 1];
  if (threadIdx.x == 0) gauss_weights(w);
  __syncthreads();
  const MaskDet& dt = dets[blockIdx.y];
  const int ew = dt.ext[2] - dt.ext[0], eh = dt.ext[3] - dt.ext[1], bw = dt.box[2] - dt.box[0];
  const int t = blockIdx.x * kScene + threadIdx.x;
  if (ew <= 0 || eh <= 0 || t >= ew * eh) return;
  const int v = dt.ext[1] + t / ew, u = dt.ext[0] + t % ew;
  const float* d = depth + (size_t)dt.frame * H * W;
  const uint8_t* m = tiles + dt.tile;
  float sn = 0.f, sd = 0.f;
  for (int k = -kRadius; k <= kRadius; ++k) {
    const int r = reflect(v + k, H);
    if (!in_box(dt.box, u, r) || !m[(size_t)(r - dt.box[1]) * bw + (u - dt.box[0])]) continue;
    const float z = d[(size_t)r * W + u];
    if (z > 0.f) { sn = __fadd_rn(sn, __fmul_rn(w[k + kRadius], z)); sd = __fadd_rn(sd, w[k + kRadius]); }
  }
  num[dt.ext_off + t] = sn;
  den[dt.ext_off + t] = sd;
}

// pass 2, along u: S = (G_u * num) / (G_u * den); columns outside the ext tile hold num = den = 0 and add +0
__global__ void __launch_bounds__(kScene)
masked_smooth_u_kernel(int W, const MaskDet* __restrict__ dets, const float* __restrict__ num,
                       const float* __restrict__ den, float* __restrict__ S) {
  __shared__ float w[2 * kRadius + 1];
  if (threadIdx.x == 0) gauss_weights(w);
  __syncthreads();
  const MaskDet& dt = dets[blockIdx.y];
  const int ew = dt.ext[2] - dt.ext[0], eh = dt.ext[3] - dt.ext[1];
  const int t = blockIdx.x * kScene + threadIdx.x;
  if (ew <= 0 || eh <= 0 || t >= ew * eh) return;
  const int row = t / ew, u = dt.ext[0] + t % ew;
  const float* a = num + dt.ext_off + (size_t)row * ew;
  const float* b = den + dt.ext_off + (size_t)row * ew;
  float sn = 0.f, sd = 0.f;
  for (int k = -kRadius; k <= kRadius; ++k) {
    const int j = reflect(u + k, W);
    if (j < dt.ext[0] || j >= dt.ext[2]) continue;
    sn = __fadd_rn(sn, __fmul_rn(w[k + kRadius], a[j - dt.ext[0]]));
    sd = __fadd_rn(sd, __fmul_rn(w[k + kRadius], b[j - dt.ext[0]]));
  }
  S[dt.ext_off + t] = sd > 0.f ? __fdiv_rn(sn, sd) : 0.f;
}

// the map over the box: gradients of the ext tile at frame indices (stencils stay inside ext by kMargin)
__global__ void __launch_bounds__(kScene)
masked_normals_kernel(int H, int W, const MaskDet* __restrict__ dets, const float* __restrict__ depth,
                      const float* __restrict__ Kmat, float lo, float hi, const float* __restrict__ S,
                      float* __restrict__ map) {
  const MaskDet& dt = dets[blockIdx.y];
  const int bw = dt.box[2] - dt.box[0], bh = dt.box[3] - dt.box[1], ew = dt.ext[2] - dt.ext[0];
  const int t = blockIdx.x * kScene + threadIdx.x;
  if (bw <= 0 || bh <= 0 || t >= bw * bh) return;
  const int v = dt.box[1] + t / bw, u = dt.box[0] + t % bw;
  const float* s = S + dt.ext_off;
  const float* col = s + (u - dt.ext[0]);                       // column u from frame row ext[1]
  const float* row = s + (size_t)(v - dt.ext[1]) * ew;           // row v from frame column ext[0]
  const float gv = gradient2(col, v, H, ew, dt.ext[1]), gu = gradient2(row, u, W, 1, dt.ext[0]);
  map_entry(u, v, Kmat + 9 * dt.frame, row[u - dt.ext[0]], gu, gv, depth[(size_t)dt.frame * H * W + (size_t)v * W + u], lo, hi,
            map + (dt.tile + t) * 6);
}

struct HypWork {   // per-hypothesis slices of the workspace, H * W entries each
  int* src;        // compacted source pixel indices
  unsigned* dist;  // pair distance bits of the current iteration (kNoPair: none)
  int* tgt;        // target pixel index of the pair
};

__device__ __forceinline__ double warp_sum(double x) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
  return x;
}

// fixed-order block sum of n doubles per thread into red[0..n): shuffle tree, then the warps in order by thread j
template <int N>
__device__ void block_sum(double (&v)[N], double* red_warp, double* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < N; ++j) {
    const double s = warp_sum(v[j]);
    if (lane == 0) red_warp[warp * N + j] = s;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    double s = 0.0;
    for (int w = 0; w < kWarps; ++w) s += red_warp[w * N + threadIdx.x];
    red[threadIdx.x] = s;
  }
  __syncthreads();
}

// exclusive row-major rank of this thread's flag in the block; *total = number of set flags
__device__ __forceinline__ int block_rank(bool flag, int* warp_counts, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ballot = __ballot_sync(0xffffffffu, flag);
  if (lane == 0) warp_counts[warp] = __popc(ballot);
  __syncthreads();
  int before = 0, all = 0;
  for (int w = 0; w < kWarps; ++w) { const int c = warp_counts[w]; before += w < warp ? c : 0; all += c; }
  __syncthreads();
  *total = all;
  return before + __popc(ballot & ((1u << lane) - 1u));
}

struct SelectShared {      // scratch of radix_select
  int hist[256];
  unsigned prefix;
  int rank;
};

// Exact select over the float bits of n distances (kNoPair entries are skipped): every thread of the CTA calls it with
// the same arguments and gets the bits of the element of rank `rank` (0-based, ascending) among the others.  Radix
// select, 8 bits per pass from the top byte; for non-negative floats the bit order is the value order.  `rank` must be
// below the number of entries that are not kNoPair.
__device__ unsigned radix_select(const unsigned* bits, int n, int rank, SelectShared& s) {
  const int tid = threadIdx.x;
  if (tid == 0) { s.prefix = 0u; s.rank = rank; }
  for (int pass = 3; pass >= 0; --pass) {
    if (tid < 256) s.hist[tid] = 0;
    __syncthreads();
    const unsigned hi_mask = pass == 3 ? 0u : ~0u << (8 * (pass + 1));
    const unsigned prefix = s.prefix;
    for (int i = tid; i < n; i += kThreads) {
      const unsigned d = bits[i];
      if (d != kNoPair && (d & hi_mask) == prefix) atomicAdd(&s.hist[(d >> (8 * pass)) & 255u], 1);
    }
    __syncthreads();
    if (tid == 0) {
      int r = s.rank, b = 0;
      while (b < 255 && r >= s.hist[b]) { r -= s.hist[b]; ++b; }
      s.rank = r;
      s.prefix = prefix | ((unsigned)b << (8 * pass));
    }
    __syncthreads();
  }
  return s.prefix;
}

struct Shared {
  double red_warp[kWarps * kAcc];
  double red[kAcc];
  double dT[12];          // current correction [R | t], row-major 3 x 4
  double residual, fitness;
  float Tf[12];
  float K[4];             // fx, fy, cx, cy
  SelectShared sel;
  int warp_counts[kWarps];
  int done;               // 0 running, 1 level converged, 2 degenerate, 3 lost
  int box[4];
};

// debug trace: record `rec` of hypothesis h (thread 0 only); records past the capacity are counted, not written
__device__ void trace_write(const gp_icp_debug_t& d, int h, int rec, int level, int it, int n, int found, unsigned median,
                            const Shared& sh, bool have_sums, const double* xi) {
  if (rec < d.trace_capacity) {
    gp_icp_trace_t& t = d.trace[(size_t)h * d.trace_capacity + rec];
    t.level = level; t.iteration = it; t.n = n; t.found = found;
    t.kept = have_sums ? (int32_t)sh.red[28] : 0;
    t.done = sh.done; t.median_bits = median; t.reserved = 0;
    for (int k = 0; k < 12; ++k) { t.Tf[k] = sh.Tf[k]; t.dT[k] = sh.dT[k]; }
    for (int k = 0; k < kAcc; ++k) t.sums[k] = have_sums ? sh.red[k] : 0.0;
    for (int k = 0; k < 6; ++k) t.xi[k] = xi[k];
  }
  d.trace_count[h] = rec + 1;
}

__device__ __forceinline__ void rodrigues(const double w[3], double R[9]) {
  const double th = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
  double A, B;                                         // sin(th)/th, (1 - cos(th))/th^2
  if (th < 1e-8) { A = 1.0 - th * th / 6.0; B = 0.5 - th * th / 24.0; }
  else { A = sin(th) / th; B = (1.0 - cos(th)) / (th * th); }
  const double x = w[0], y = w[1], z = w[2];
  R[0] = 1.0 - B * (y * y + z * z); R[1] = -A * z + B * x * y;     R[2] = A * y + B * x * z;
  R[3] = A * z + B * x * y;         R[4] = 1.0 - B * (x * x + z * z); R[5] = -A * x + B * y * z;
  R[6] = -A * y + B * x * z;        R[7] = A * x + B * y * z;     R[8] = 1.0 - B * (x * x + y * y);
}

// kBox = false: frame maps [n_frames,H,W,6], frame_idx [n_hyp] and optional full-frame masks [n_hyp,H,W] (stages 1-2).
// kBox = true: the masked mode (1'-2'): frame_idx is det_idx [n_hyp] into the n_frames entries of `dets`, the map and
// mask are the detection's box tiles, and the per-hypothesis scratch holds `scratch` entries (>= every box area).
template <bool kBox>
__global__ void __launch_bounds__(kThreads, 1)
icp_kernel(int n_frames, int H, int W, const int32_t* __restrict__ frame_idx, const uint8_t* __restrict__ masks,
           const float* __restrict__ rendered, const int64_t* __restrict__ boxes, const float* __restrict__ T0,
           const float* __restrict__ Kmat, const float* __restrict__ map, gp_icp_params_t p, int* src_all,
           unsigned* dist_all, int* tgt_all, float* __restrict__ out_pose, int32_t* __restrict__ out_status,
           float* __restrict__ out_residual, float* __restrict__ out_fitness, const MaskDet* __restrict__ dets,
           long long scratch) {
  __shared__ Shared sh;
  const int h = blockIdx.x, tid = threadIdx.x;
  const size_t plane = (size_t)H * W;
  const bool trace = p.debug.trace != nullptr;
  int n_rec = 0;                                       // trace records of this hypothesis (thread 0)
  if (tid == 0 && p.debug.trace_count) p.debug.trace_count[h] = 0;
  const float* t0 = T0 + 16 * (size_t)h;
  const float upm = p.unit_per_m;
  float* po = out_pose + 16 * (size_t)h;
  auto keep_T0 = [&](int status, float res, float fit) {
    if (tid < 16) po[tid] = t0[tid];
    if (tid == 0) { out_status[h] = status; out_residual[h] = res; out_fitness[h] = fit; }
  };
  const int fi = frame_idx[h];
  if (fi < 0 || fi >= n_frames) { keep_T0(GP_ICP_INVALID, -1.f, 0.f); return; }
  // target region: the frame, or the mask box (tb) with box-relative map and mask tiles
  int tb[4] = {0, 0, W, H};
  if (kBox) {
    for (int k = 0; k < 4; ++k) tb[k] = dets[fi].box[k];
    if (tb[2] < tb[0]) tb[2] = tb[0];
    if (tb[3] < tb[1]) tb[3] = tb[1];
    if ((long long)(tb[2] - tb[0]) * (tb[3] - tb[1]) > scratch) { keep_T0(GP_ICP_INVALID, -1.f, 0.f); return; }
  }
  const int f = kBox ? dets[fi].frame : fi, tw = tb[2] - tb[0];
  const size_t stride = kBox ? (size_t)scratch : plane;
  HypWork wk{src_all + h * stride, dist_all + h * stride, tgt_all + h * stride};
  const float* R = rendered + h * plane;
  const float* M = kBox ? map + dets[fi].tile * 6 : map + f * plane * 6;
  const uint8_t* mask = kBox ? masks + dets[fi].tile : masks ? masks + h * plane : nullptr;
  const float delta = __fmul_rn(0.1f, upm);
  auto entry = [&](int u, int v) -> size_t {          // map / mask entry of frame pixel (u, v) inside tb
    return kBox ? (size_t)(v - tb[1]) * tw + (u - tb[0]) : (size_t)v * W + u;
  };
  if (tid == 0) {
    const float* K = Kmat + 9 * f;
    sh.K[0] = K[0]; sh.K[1] = K[4]; sh.K[2] = K[2]; sh.K[3] = K[5];
    const int64_t* b = boxes + 4 * (size_t)h;
    sh.box[0] = (int)max((int64_t)0, min((int64_t)W, b[0])); sh.box[1] = (int)max((int64_t)0, min((int64_t)H, b[1]));
    sh.box[2] = (int)max((int64_t)0, min((int64_t)W, b[2])); sh.box[3] = (int)max((int64_t)0, min((int64_t)H, b[3]));
  }
  __syncthreads();
  const float fx = sh.K[0], fy = sh.K[1], cx = sh.K[2], cy = sh.K[3];
  auto target_ok = [&](int u, int v) -> bool {
    const size_t e = entry(u, v);
    const float d = M[e * 6 + 2];
    if (!(d > 0.f)) return false;
    if (mask) return mask[e] != 0;
    const float r = R[(size_t)v * W + u];
    return r > 0.f && fabsf(__fsub_rn(d, r)) <= delta;
  };

  // stages 2-4: counts and centroids of both sets, sources compacted in row-major order inside the box
  const int bx0 = sh.box[0], by0 = sh.box[1], bw = sh.box[2] - sh.box[0], bh = sh.box[3] - sh.box[1];
  const int rx0 = mask ? tb[0] : bx0, ry0 = mask ? tb[1] : by0, rw = mask ? tw : max(bw, 0);
  const int rh = mask ? tb[3] - tb[1] : max(bh, 0);
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};            // targets: n, x, y, z; sources: x, y, z
  int nsrc = 0;
  const int region = rw * rh;
  for (int base = 0; base < region; base += kThreads) {
    const int i = base + tid;
    bool is_src = false;
    if (i < region) {
      const int v = ry0 + i / rw, u = rx0 + i % rw;
      const size_t q = (size_t)v * W + u, e = entry(u, v);
      if (target_ok(u, v)) {
        acc[0] += 1.0; acc[1] += M[e * 6]; acc[2] += M[e * 6 + 1]; acc[3] += M[e * 6 + 2];
        const float r = R[q];
        if (r > 0.f && u >= bx0 && u < bx0 + bw && v >= by0 && v < by0 + bh) {
          is_src = true;
          acc[4] += __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), r), fx);
          acc[5] += __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), r), fy);
          acc[6] += r;
        }
      }
    }
    int total;
    const int rank = block_rank(is_src, sh.warp_counts, &total);
    if (is_src) wk.src[nsrc + rank] = (ry0 + i / rw) * W + rx0 + i % rw;
    nsrc += total;
  }
  block_sum(acc, sh.red_warp, sh.red);
  const int ntgt = (int)sh.red[0];
  if (ntgt < p.min_points || nsrc < p.min_points) { keep_T0(GP_ICP_TOO_FEW_POINTS, -1.f, 0.f); return; }
  if (tid == 0) {
    for (int k = 0; k < 12; ++k) sh.dT[k] = (k % 4 == k / 4) ? 1.0 : 0.0;
    for (int k = 0; k < 3; ++k) sh.dT[4 * k + 3] = sh.red[1 + k] / ntgt - sh.red[4 + k] / nsrc;
    if (p.debug.pose0)
      for (int k = 0; k < 12; ++k) p.debug.pose0[12 * (size_t)h + k] = (float)sh.dT[k];
    if (p.debug.counts) { p.debug.counts[2 * h] = ntgt; p.debug.counts[2 * h + 1] = nsrc; }
  }
  if (p.debug.sources)
    for (int i = tid; i < nsrc; i += kThreads) p.debug.sources[h * plane + i] = wk.src[i];

  const double L = (double)upm;
  const float gate_step_t = __fmul_rn(p.min_step_m, upm);
  if (tid == 0) { sh.residual = -1.0; sh.fitness = 0.0; }
  __syncthreads();                                     // sh.dT, sh.residual and sh.fitness are read by every thread
  int status = GP_ICP_OK;
  for (int level = p.num_levels - 1; level >= 0 && status == GP_ICP_OK; --level) {
    const int stride = 1 << level, n = (nsrc + stride - 1) >> level, rad = 2 << level;
    int it = 0;
    for (; it < p.max_iters; ++it) {
      if (tid < 12) sh.Tf[tid] = (float)sh.dT[tid];
      __syncthreads();
      float T[12];
#pragma unroll
      for (int k = 0; k < 12; ++k) T[k] = sh.Tf[k];
      // association
      int found = 0;
      for (int i = tid; i < n; i += kThreads) {
        const int q = wk.src[i * stride];
        const int v = q / W, u = q - v * W;
        const float z = R[q];
        const float x = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), z), fx);
        const float y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), z), fy);
        float s[3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
          s[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], x), __fmul_rn(T[4 * r + 1], y)),
                                     __fmul_rn(T[4 * r + 2], z)), T[4 * r + 3]);
        unsigned best = kNoPair;
        int bi = -1;
        if (s[2] > 0.f) {
          const float pu = __fadd_rn(__fdiv_rn(__fmul_rn(fx, s[0]), s[2]), cx);
          const float pv = __fadd_rn(__fdiv_rn(__fmul_rn(fy, s[1]), s[2]), cy);
          if (fabsf(pu) < 1e7f && fabsf(pv) < 1e7f) {
            const int cu = (int)rintf(pu), cv = (int)rintf(pv);
            const int u0 = max(cu - rad, tb[0]), u1 = min(cu + rad, tb[2] - 1);
            const int v0 = max(cv - rad, tb[1]), v1 = min(cv + rad, tb[3] - 1);
            float bd = 0.f;
            for (int vv = v0; vv <= v1; ++vv)
              for (int uu = u0; uu <= u1; ++uu) {
                if (!target_ok(uu, vv)) continue;
                const size_t t = (size_t)vv * W + uu, e = entry(uu, vv);
                const float dx = __fsub_rn(M[e * 6], s[0]), dy = __fsub_rn(M[e * 6 + 1], s[1]);
                const float dz = __fsub_rn(M[e * 6 + 2], s[2]);
                const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                if (bi < 0 || d2 < bd) { bd = d2; bi = (int)t; }
              }
            const float dist = __fsqrt_rn(bd);
            if (bi >= 0 && dist < __uint_as_float(kNoPair)) best = __float_as_uint(dist);
            else bi = -1;                              // a distance that overflowed (or NaN) is no pair
          }
        }
        wk.dist[i] = best;
        wk.tgt[i] = bi;
        found += bi >= 0;
      }
      // exact median: the element of rank (m - 1) / 2 of the m pair distances
      double m_[1] = {(double)found};
      block_sum(m_, sh.red_warp, sh.red);
      const int total = (int)sh.red[0];
      if (total == 0) {
        if (trace && tid == 0) {
          const double zero[6] = {0, 0, 0, 0, 0, 0};
          sh.done = 3;
          trace_write(p.debug, h, n_rec++, level, it, n, 0, kNoPair, sh, false, zero);
        }
        status = GP_ICP_LOST;
        break;
      }
      const unsigned median = radix_select(wk.dist, n, (total - 1) / 2, sh.sel);
      const float gate = __fmul_rn(p.rejection_scale, __uint_as_float(median));
      // normal equations
      double a[kAcc];
#pragma unroll
      for (int k = 0; k < kAcc; ++k) a[k] = 0.0;
      const bool last_level = level == 0;
      for (int i = tid; i < n; i += kThreads) {
        const int t = wk.tgt[i];
        const unsigned db = wk.dist[i];
        const bool kept = t >= 0 && __uint_as_float(db) <= gate;
        if (last_level && p.debug.assoc) p.debug.assoc[h * plane + i] = t < 0 ? -1 : kept ? t : -2 - t;
        if (!kept) continue;
        const int q = wk.src[i * stride];
        const int v = q / W, u = q - v * W;
        const float z = R[q];
        const float x = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), z), fx);
        const float y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), z), fy);
        double s[3];
#pragma unroll
        for (int r = 0; r < 3; ++r)
          s[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(T[4 * r], x), __fmul_rn(T[4 * r + 1], y)),
                                     __fmul_rn(T[4 * r + 2], z)), T[4 * r + 3]);
        const float* tm = M + (kBox ? entry(t % W, t / W) : (size_t)t) * 6;
        const double nx = tm[3], ny = tm[4], nz = tm[5];
        const double r = (s[0] - tm[0]) * nx + (s[1] - tm[1]) * ny + (s[2] - tm[2]) * nz;
        const double j[6] = {(s[1] * nz - s[2] * ny) / L, (s[2] * nx - s[0] * nz) / L, (s[0] * ny - s[1] * nx) / L,
                             nx, ny, nz};
        int k = 0;
#pragma unroll
        for (int c = 0; c < 6; ++c)
#pragma unroll
          for (int e = c; e < 6; ++e) a[k++] += j[c] * j[e];
#pragma unroll
        for (int c = 0; c < 6; ++c) a[21 + c] += j[c] * r;
        a[27] += r * r;
        a[28] += 1.0;
      }
      block_sum(a, sh.red_warp, sh.red);
      if (tid == 0) {
        const double* S = sh.red;
        const double kept = S[28];
        if (last_level) { sh.residual = kept > 0 ? sqrt(S[27] / kept) : -1.0; sh.fitness = kept / n; }
        double A[6][6], b[6], dmax = 0.0;
        int k = 0;
        for (int c = 0; c < 6; ++c)
          for (int e = c; e < 6; ++e) { A[c][e] = A[e][c] = S[k++]; }
        for (int c = 0; c < 6; ++c) { b[c] = -S[21 + c]; dmax = fmax(dmax, A[c][c]); }
        bool ok = true;
        for (int c = 0; c < 6 && ok; ++c) {          // in-place Cholesky, A = L L^T
          double d = A[c][c];
          for (int e = 0; e < c; ++e) d -= A[c][e] * A[c][e];
          if (!(d > 1e-8 * dmax)) { ok = false; break; }
          A[c][c] = sqrt(d);
          for (int r = c + 1; r < 6; ++r) {
            double s = A[r][c];
            for (int e = 0; e < c; ++e) s -= A[r][e] * A[c][e];
            A[r][c] = s / A[c][c];
          }
        }
        double xi[6] = {0, 0, 0, 0, 0, 0};
        if (kept < 6.0) {
          sh.done = 3;
        } else if (!ok) {
          sh.done = 2;
        } else {
          double y[6];
          for (int c = 0; c < 6; ++c) {
            double s = b[c];
            for (int e = 0; e < c; ++e) s -= A[c][e] * y[e];
            y[c] = s / A[c][c];
          }
          for (int c = 5; c >= 0; --c) {
            double s = y[c];
            for (int e = c + 1; e < 6; ++e) s -= A[e][c] * xi[e];
            xi[c] = s / A[c][c];
          }
          const double w[3] = {xi[0] / L, xi[1] / L, xi[2] / L};
          double Rw[9], N[12];
          rodrigues(w, Rw);
          for (int r = 0; r < 3; ++r)
            for (int c = 0; c < 4; ++c)
              N[4 * r + c] = Rw[3 * r] * sh.dT[c] + Rw[3 * r + 1] * sh.dT[4 + c] + Rw[3 * r + 2] * sh.dT[8 + c] +
                             (c == 3 ? xi[3 + r] : 0.0);
          for (int c = 0; c < 12; ++c) sh.dT[c] = N[c];
          const double wn = sqrt(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
          const double vn = sqrt(xi[3] * xi[3] + xi[4] * xi[4] + xi[5] * xi[5]);
          sh.done = (wn < p.min_step_rad && vn < gate_step_t) ? 1 : 0;
        }
        if (trace) trace_write(p.debug, h, n_rec++, level, it, n, total, median, sh, true, xi);
      }
      __syncthreads();
      const int done = sh.done;
      __syncthreads();
      if (done == 2) { status = GP_ICP_DEGENERATE; break; }
      if (done == 3) { status = GP_ICP_LOST; break; }
      if (done == 1) { ++it; break; }
    }
    if (p.debug.iterations && tid == 0) p.debug.iterations[(size_t)h * p.num_levels + level] = it;
  }
  __syncthreads();
  const double residual = sh.residual, fitness = sh.fitness;
  if (status == GP_ICP_OK && !(residual >= 0.0 && residual <= (double)__fmul_rn(p.max_residual, upm)))
    status = GP_ICP_RESIDUAL;
  if (status != GP_ICP_OK) {
    keep_T0(status, (float)residual, (float)fitness);
    return;
  }
  if (tid < 12) {                                      // (dT T0)[r][c]; T0's last row is (0, 0, 0, 1)
    const int r = tid / 4, c = tid % 4;
    po[tid] = (float)(sh.dT[4 * r] * t0[c] + sh.dT[4 * r + 1] * t0[4 + c] + sh.dT[4 * r + 2] * t0[8 + c] +
                      (c == 3 ? sh.dT[4 * r + 3] : 0.0));
  } else if (tid < 16) {
    po[tid] = t0[tid];
  }
  if (tid == 0) { out_status[h] = GP_ICP_OK; out_residual[h] = (float)residual; out_fitness[h] = (float)fitness; }
}

// gp_debug_icp_select: out[0] = m, the entries that are not kNoPair; out[1] = radix_select's element of rank `rank`
// among them (kNoPair when rank >= m)
__global__ void __launch_bounds__(kThreads, 1)
select_kernel(const unsigned* __restrict__ bits, int n, int rank, unsigned* __restrict__ out) {
  __shared__ SelectShared sel;
  __shared__ int count;
  if (threadIdx.x == 0) count = 0;
  __syncthreads();
  int c = 0;
  for (int i = threadIdx.x; i < n; i += kThreads) c += bits[i] != kNoPair;
  atomicAdd(&count, c);
  __syncthreads();
  const int m = count;
  const unsigned v = rank < m ? radix_select(bits, n, rank, sel) : kNoPair;
  if (threadIdx.x == 0) { out[0] = (unsigned)m; out[1] = v; }
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

size_t scene_bytes(int n_frames, int H, int W) { return align256((size_t)n_frames * H * W * 9 * sizeof(float)); }

int check_sizes(int n_frames, int n_hyp, int H, int W) {
  if (n_frames < 1 || n_frames > 65535) return fail(GP_ERR_INVALID, "n_frames %d outside [1, 65535]", n_frames);
  if (n_hyp < 0 || n_hyp > 65535) return fail(GP_ERR_INVALID, "n_hyp %d outside [0, 65535]", n_hyp);
  if (H < kMinSide || W < kMinSide || H > kMaxSide || W > kMaxSide)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [%d, %d]", H, W, kMinSide, kMaxSide);
  return GP_OK;
}

int check_params(const gp_icp_params_t* params) {
  if (!params) return fail(GP_ERR_INVALID, "null params");
  const gp_icp_params_t& p = *params;
  if (!(p.unit_per_m > 0.f) || !isfinite(p.unit_per_m))
    return fail(GP_ERR_INVALID, "unit_per_m must be positive and finite");
  if (p.min_points < 1) return fail(GP_ERR_INVALID, "min_points %d must be >= 1", p.min_points);
  if (p.num_levels < 1 || p.num_levels > kMaxLevels)
    return fail(GP_ERR_INVALID, "num_levels %d outside [1, %d]", p.num_levels, kMaxLevels);
  if (p.max_iters < 1 || p.max_iters > 100000) return fail(GP_ERR_INVALID, "max_iters %d outside [1, 100000]", p.max_iters);
  if (!(p.rejection_scale > 0.f) || !isfinite(p.rejection_scale))
    return fail(GP_ERR_INVALID, "rejection_scale must be positive and finite");
  if (!(p.max_residual >= 0.f) || !(p.min_step_rad >= 0.f) || !(p.min_step_m >= 0.f))
    return fail(GP_ERR_INVALID, "max_residual, min_step_rad and min_step_m must be >= 0");
  if (p.debug.trace && (p.debug.trace_capacity < 1 || !p.debug.trace_count))
    return fail(GP_ERR_INVALID, "debug.trace needs trace_capacity >= 1 and trace_count");
  return GP_OK;
}

// the masked workspace: the detection table, then the mask tiles, the map, num, den, S and the run ends
struct MaskLayout {
  std::vector<MaskDet> dets;
  long long tiles = 0, exts = 0, box_max = 0, ext_max = 0, runs = 0;
  size_t table_b = 0, tiles_b = 0, map_b = 0, ext_b = 0, ends_b = 0;
  size_t bytes() const { return table_b + tiles_b + map_b + 3 * ext_b + ends_b; }
};

int mask_layout(int n_frames, int H, int W, const gp_icp_mask_set_t* set, MaskLayout* L) {
  if (const int rc = check_sizes(n_frames, 0, H, W)) return rc;
  if (!set) return fail(GP_ERR_INVALID, "null mask set");
  const int n = set->n_det;
  if (n < 0 || n > 65535) return fail(GP_ERR_INVALID, "n_det %d outside [0, 65535]", n);
  if (n && (!set->frame || !set->boxes)) return fail(GP_ERR_INVALID, "null frame / boxes");
  const int64_t* ro = set->run_offsets;
  if (ro && ro[0] < 0) return fail(GP_ERR_INVALID, "run_offsets[0] = %lld is negative", (long long)ro[0]);
  L->dets.resize(n);
  for (int d = 0; d < n; ++d) {
    const int32_t* b = set->boxes + 4 * (size_t)d;
    if (set->frame[d] < 0 || set->frame[d] >= n_frames)
      return fail(GP_ERR_INVALID, "frame[%d] = %d outside [0, %d)", d, set->frame[d], n_frames);
    if (b[0] < 0 || b[0] > b[2] || b[2] > W || b[1] < 0 || b[1] > b[3] || b[3] > H)
      return fail(GP_ERR_INVALID, "box %d (%d, %d, %d, %d) is not 0 <= x0 <= x1 <= %d, 0 <= y0 <= y1 <= %d", d, b[0],
                  b[1], b[2], b[3], W, H);
    if (ro && ro[d + 1] < ro[d])
      return fail(GP_ERR_INVALID, "run_offsets decrease at detection %d (%lld -> %lld)", d, (long long)ro[d],
                  (long long)ro[d + 1]);
    MaskDet& m = L->dets[d];
    const bool empty = b[0] == b[2] || b[1] == b[3];
    for (int k = 0; k < 4; ++k) m.box[k] = b[k];
    m.ext[0] = empty ? b[0] : max(0, b[0] - kMargin); m.ext[1] = empty ? b[1] : max(0, b[1] - kMargin);
    m.ext[2] = empty ? b[0] : min(W, b[2] + kMargin); m.ext[3] = empty ? b[1] : min(H, b[3] + kMargin);
    m.frame = set->frame[d];
    m.reserved = 0;
    m.tile = L->tiles;
    m.ext_off = L->exts;
    m.run0 = ro ? ro[d] : 0;
    m.run1 = ro ? ro[d + 1] : 0;
    const long long area = (long long)(b[2] - b[0]) * (b[3] - b[1]);
    const long long ext = (long long)(m.ext[2] - m.ext[0]) * (m.ext[3] - m.ext[1]);
    L->tiles += area;
    L->exts += ext;
    L->box_max = std::max(L->box_max, area);
    L->ext_max = std::max(L->ext_max, ext);
  }
  L->runs = ro ? ro[n] : 0;
  L->table_b = align256((size_t)n * sizeof(MaskDet));
  L->tiles_b = align256((size_t)L->tiles);
  L->map_b = align256((size_t)L->tiles * 6 * sizeof(float));
  L->ext_b = align256((size_t)L->exts * sizeof(float));
  L->ends_b = align256((size_t)L->runs * sizeof(long long));
  return GP_OK;
}

struct MaskPtrs {
  MaskDet* dets;
  uint8_t* tiles;
  float *map, *num, *den, *S;
  long long* ends;
};

MaskPtrs mask_ptrs(const MaskLayout& L, void* workspace) {
  char* w = static_cast<char*>(workspace);
  MaskPtrs p;
  p.dets = reinterpret_cast<MaskDet*>(w);
  p.tiles = reinterpret_cast<uint8_t*>(w += L.table_b);
  p.map = reinterpret_cast<float*>(w += L.tiles_b);
  p.num = reinterpret_cast<float*>(w += L.map_b);
  p.den = reinterpret_cast<float*>(w += L.ext_b);
  p.S = reinterpret_cast<float*>(w += L.ext_b);
  p.ends = reinterpret_cast<long long*>(w += L.ext_b);
  return p;
}

unsigned blocks(long long pixels) { return (unsigned)((pixels + kScene - 1) / kScene); }

}  // namespace

extern "C" int gp_icp_masked_query_sizes(int n_frames, int height, int width, const gp_icp_mask_set_t* set,
                                         size_t* workspace_bytes, int64_t* box_pixels, size_t* tiles_offset,
                                         size_t* map_offset) {
  MaskLayout L;
  if (const int rc = mask_layout(n_frames, height, width, set, &L)) return rc;
  if (!workspace_bytes || !box_pixels) return fail(GP_ERR_INVALID, "null workspace_bytes / box_pixels");
  *workspace_bytes = L.bytes();
  *box_pixels = L.box_max;
  if (tiles_offset) *tiles_offset = L.table_b;
  if (map_offset) *map_offset = L.table_b + L.tiles_b;
  return GP_OK;
}

extern "C" int gp_icp_masked_decode(int n_frames, int height, int width, const gp_icp_mask_set_t* set,
                                    const uint8_t* masks, const int32_t* counts, void* workspace, void* stream) {
  MaskLayout L;
  if (const int rc = mask_layout(n_frames, height, width, set, &L)) return rc;
  if (!workspace) return fail(GP_ERR_INVALID, "null workspace");
  if (!masks == !set->run_offsets) return fail(GP_ERR_INVALID, "give either dense masks or run_offsets, not both");
  if (!masks && L.runs > 0 && !counts) return fail(GP_ERR_INVALID, "null counts");
  const int n = set->n_det;
  if (n == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const MaskPtrs P = mask_ptrs(L, workspace);
  GP_CUDA(cudaMemcpyAsync(P.dets, L.dets.data(), (size_t)n * sizeof(MaskDet), cudaMemcpyHostToDevice, st));
  if (!masks && L.runs > 0) GP_CUDA(gp::launch_rle_scan(n, counts, set->run_offsets, P.ends, st));
  if (L.box_max > 0)
    GP_CUDA(gp::launch_ex(mask_tiles_kernel, dim3(blocks(L.box_max), n), kScene, 0, st, 1, false, height, width,
                          P.dets, masks, P.ends, P.tiles));
  return GP_OK;
}

extern "C" int gp_icp_prepare_masked_scene(int n_frames, int height, int width, const gp_icp_mask_set_t* set,
                                           const float* depth, const float* K, float unit_per_m, void* workspace,
                                           void* stream) {
  MaskLayout L;
  if (const int rc = mask_layout(n_frames, height, width, set, &L)) return rc;
  if (!depth || !K || !workspace) return fail(GP_ERR_INVALID, "null argument");
  if (!(unit_per_m > 0.f) || !isfinite(unit_per_m))
    return fail(GP_ERR_INVALID, "unit_per_m must be positive and finite");
  const int n = set->n_det;
  if (n == 0 || L.box_max == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const MaskPtrs P = mask_ptrs(L, workspace);
  const dim3 ge(blocks(L.ext_max), n), gb(blocks(L.box_max), n);
  GP_CUDA(gp::launch_ex(masked_smooth_v_kernel, ge, kScene, 0, st, 1, false, height, width, P.dets, depth, P.tiles,
                        P.num, P.den));
  GP_CUDA(gp::launch_ex(masked_smooth_u_kernel, ge, kScene, 0, st, 1, false, width, P.dets, P.num, P.den, P.S));
  GP_CUDA(gp::launch_ex(masked_normals_kernel, gb, kScene, 0, st, 1, false, height, width, P.dets, depth, K,
                        0.2f * unit_per_m, 5.f * unit_per_m, P.S, P.map));
  return GP_OK;
}

extern "C" int gp_icp_refine_masked(int n_frames, int height, int width, const gp_icp_mask_set_t* set, int n_hyp,
                                    const int32_t* det_idx, const float* rendered_depth, const int64_t* boxes,
                                    const float* T0, const float* K, const gp_icp_params_t* params, float* out_poses,
                                    int32_t* out_status, float* out_residual, float* out_fitness,
                                    const void* scene_workspace, void* workspace, void* stream) {
  MaskLayout L;
  if (const int rc = mask_layout(n_frames, height, width, set, &L)) return rc;
  if (const int rc = check_sizes(n_frames, n_hyp, height, width)) return rc;
  if (const int rc = check_params(params)) return rc;
  if (!det_idx || !rendered_depth || !boxes || !T0 || !K || !out_poses || !out_status || !out_residual ||
      !out_fitness || !scene_workspace || (!workspace && L.box_max > 0))
    return fail(GP_ERR_INVALID, "null argument");
  if (n_hyp == 0) return GP_OK;
  const size_t per = (size_t)n_hyp * L.box_max;
  int* src = static_cast<int*>(workspace);
  unsigned* dist = reinterpret_cast<unsigned*>(src + per);
  int* tgt = reinterpret_cast<int*>(dist + per);
  const MaskPtrs P = mask_ptrs(L, const_cast<void*>(scene_workspace));
  GP_CUDA(gp::launch_ex(icp_kernel<true>, n_hyp, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false, set->n_det,
                        height, width, det_idx, P.tiles, rendered_depth, boxes, T0, K, P.map, *params, src, dist, tgt,
                        out_poses, out_status, out_residual, out_fitness, P.dets, L.box_max));
  return GP_OK;
}

extern "C" int gp_icp_query_sizes(int n_frames, int n_hyp, int height, int width, size_t* workspace_bytes) {
  if (const int rc = check_sizes(n_frames, n_hyp, height, width)) return rc;
  if (!workspace_bytes) return fail(GP_ERR_INVALID, "null workspace_bytes");
  *workspace_bytes = scene_bytes(n_frames, height, width) + (size_t)n_hyp * height * width * 3 * sizeof(int);
  return GP_OK;
}

extern "C" int gp_icp_prepare_scene(int n_frames, int height, int width, const float* depth, const float* K,
                                    float unit_per_m, void* workspace, void* stream) {
  if (const int rc = check_sizes(n_frames, 0, height, width)) return rc;
  if (!depth || !K || !workspace) return fail(GP_ERR_INVALID, "null argument");
  if (!(unit_per_m > 0.f) || !isfinite(unit_per_m))
    return fail(GP_ERR_INVALID, "unit_per_m must be positive and finite");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)n_frames * height * width;
  float* map = static_cast<float*>(workspace);
  float* num = map + plane * 6;
  float* den = num + plane;
  float* S = den + plane;
  const dim3 grid((height * width + kScene - 1) / kScene, n_frames);
  GP_CUDA(gp::launch_ex(smooth_v_kernel, grid, kScene, 0, st, 1, false, height, width, depth, num, den));
  GP_CUDA(gp::launch_ex(smooth_u_kernel, grid, kScene, 0, st, 1, false, height, width, num, den, S));
  GP_CUDA(gp::launch_ex(normals_kernel, grid, kScene, 0, st, 1, false, height, width, depth, K, 0.2f * unit_per_m,
                        5.f * unit_per_m, S, map));
  return GP_OK;
}

extern "C" int gp_icp_refine(int n_frames, int n_hyp, int height, int width, const int32_t* frame_idx,
                             const uint8_t* masks, const float* rendered_depth, const int64_t* boxes, const float* T0,
                             const float* K, const gp_icp_params_t* params, float* out_poses, int32_t* out_status,
                             float* out_residual, float* out_fitness, void* workspace, void* stream) {
  if (const int rc = check_sizes(n_frames, n_hyp, height, width)) return rc;
  if (const int rc = check_params(params)) return rc;
  const gp_icp_params_t& p = *params;
  if (!frame_idx || !rendered_depth || !boxes || !T0 || !K || !out_poses || !out_status || !out_residual ||
      !out_fitness || !workspace)
    return fail(GP_ERR_INVALID, "null argument");
  if (n_hyp == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)height * width;
  char* ws = static_cast<char*>(workspace);
  const float* map = reinterpret_cast<const float*>(ws);
  int* src = reinterpret_cast<int*>(ws + scene_bytes(n_frames, height, width));
  unsigned* dist = reinterpret_cast<unsigned*>(src + n_hyp * plane);
  int* tgt = reinterpret_cast<int*>(dist + n_hyp * plane);
  GP_CUDA(gp::launch_ex(icp_kernel<false>, n_hyp, kThreads, 0, st, 1, false, n_frames, height, width, frame_idx, masks,
                        rendered_depth, boxes, T0, K, map, p, src, dist, tgt, out_poses, out_status, out_residual,
                        out_fitness, nullptr, 0LL));
  return GP_OK;
}

extern "C" int gp_debug_icp_select(const uint32_t* bits, int n, int rank, uint32_t* out, void* stream) {
  if (n < 1) return fail(GP_ERR_INVALID, "n %d must be >= 1", n);
  if (rank < 0 || rank >= n) return fail(GP_ERR_INVALID, "rank %d outside [0, n = %d)", rank, n);
  if (!bits || !out) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(select_kernel, 1, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false, bits, n, rank, out));
  return GP_OK;
}
