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
// Debug hooks (tests/test_gpu_icp_solver.py): with debug.trace set, thread 0 writes one gp_icp_trace_t per iteration
// (the fp32 transform it associated with, the counts, the median, the 29 fp64 sums, the step and the correction after
// it), so that each step can be checked against an fp64 reference started from the kernel's own state; the outputs are
// the same with and without it.  gp_debug_icp_select runs the median's radix_select alone.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

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
__device__ __forceinline__ float gradient2(const float* x, int i, int n, int st) {
  if (i == 0)
    return __fadd_rn(__fadd_rn(__fmul_rn(-0.75f, x[0]), x[st]), __fmul_rn(-0.25f, x[2 * st]));
  if (i == n - 1)
    return __fadd_rn(__fadd_rn(__fmul_rn(0.25f, x[(size_t)(n - 3) * st]), -x[(size_t)(n - 2) * st]),
                     __fmul_rn(0.75f, x[(size_t)(n - 1) * st]));
  return __fdiv_rn(__fsub_rn(x[(size_t)(i + 1) * st], x[(size_t)(i - 1) * st]), 4.f);
}

__global__ void __launch_bounds__(kScene)
normals_kernel(int H, int W, const float* __restrict__ depth, const float* __restrict__ Kmat, float lo, float hi,
               const float* __restrict__ S, float* __restrict__ map) {
  const size_t plane = (size_t)H * W;
  const int pix = blockIdx.x * kScene + threadIdx.x, f = blockIdx.y;
  if (pix >= H * W) return;
  const int v = pix / W, u = pix - v * W;
  const float* K = Kmat + 9 * f;
  const float fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  const float* s = S + f * plane;
  const float z = s[pix];
  const float gv = gradient2(s + u, v, H, W), gu = gradient2(s + (size_t)v * W, u, W, 1);
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
  const float d = depth[f * plane + pix];
  const bool ok = d > lo && d < hi;
  float* m = map + (f * plane + pix) * 6;
  m[0] = ok ? __fdiv_rn(__fmul_rn(a, d), fx) : 0.f;
  m[1] = ok ? __fdiv_rn(__fmul_rn(b, d), fy) : 0.f;
  m[2] = ok ? d : 0.f;
  m[3] = nx; m[4] = ny; m[5] = nz;
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

__global__ void __launch_bounds__(kThreads, 1)
icp_kernel(int n_frames, int H, int W, const int32_t* __restrict__ frame_idx, const uint8_t* __restrict__ masks,
           const float* __restrict__ rendered, const int64_t* __restrict__ boxes, const float* __restrict__ T0,
           const float* __restrict__ Kmat, const float* __restrict__ map, gp_icp_params_t p, int* src_all,
           unsigned* dist_all, int* tgt_all, float* __restrict__ out_pose, int32_t* __restrict__ out_status,
           float* __restrict__ out_residual, float* __restrict__ out_fitness) {
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
  const int f = frame_idx[h];
  if (f < 0 || f >= n_frames) { keep_T0(GP_ICP_INVALID, -1.f, 0.f); return; }
  HypWork wk{src_all + h * plane, dist_all + h * plane, tgt_all + h * plane};
  const float* R = rendered + h * plane;
  const float* M = map + f * plane * 6;
  const uint8_t* mask = masks ? masks + h * plane : nullptr;
  const float delta = __fmul_rn(0.1f, upm);
  if (tid == 0) {
    const float* K = Kmat + 9 * f;
    sh.K[0] = K[0]; sh.K[1] = K[4]; sh.K[2] = K[2]; sh.K[3] = K[5];
    const int64_t* b = boxes + 4 * (size_t)h;
    sh.box[0] = (int)max((int64_t)0, min((int64_t)W, b[0])); sh.box[1] = (int)max((int64_t)0, min((int64_t)H, b[1]));
    sh.box[2] = (int)max((int64_t)0, min((int64_t)W, b[2])); sh.box[3] = (int)max((int64_t)0, min((int64_t)H, b[3]));
  }
  __syncthreads();
  const float fx = sh.K[0], fy = sh.K[1], cx = sh.K[2], cy = sh.K[3];
  auto target_ok = [&](size_t q) -> bool {
    const float d = M[q * 6 + 2];
    if (!(d > 0.f)) return false;
    if (mask) return mask[q] != 0;
    const float r = R[q];
    return r > 0.f && fabsf(__fsub_rn(d, r)) <= delta;
  };

  // stages 2-4: counts and centroids of both sets, sources compacted in row-major order inside the box
  const int bx0 = sh.box[0], by0 = sh.box[1], bw = sh.box[2] - sh.box[0], bh = sh.box[3] - sh.box[1];
  const int rx0 = mask ? 0 : bx0, ry0 = mask ? 0 : by0, rw = mask ? W : max(bw, 0), rh = mask ? H : max(bh, 0);
  double acc[7] = {0, 0, 0, 0, 0, 0, 0};            // targets: n, x, y, z; sources: x, y, z
  int nsrc = 0;
  const int region = rw * rh;
  for (int base = 0; base < region; base += kThreads) {
    const int i = base + tid;
    bool is_src = false;
    if (i < region) {
      const int v = ry0 + i / rw, u = rx0 + i % rw;
      const size_t q = (size_t)v * W + u;
      if (target_ok(q)) {
        acc[0] += 1.0; acc[1] += M[q * 6]; acc[2] += M[q * 6 + 1]; acc[3] += M[q * 6 + 2];
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
            const int u0 = max(cu - rad, 0), u1 = min(cu + rad, W - 1);
            const int v0 = max(cv - rad, 0), v1 = min(cv + rad, H - 1);
            float bd = 0.f;
            for (int vv = v0; vv <= v1; ++vv)
              for (int uu = u0; uu <= u1; ++uu) {
                const size_t t = (size_t)vv * W + uu;
                if (!target_ok(t)) continue;
                const float dx = __fsub_rn(M[t * 6], s[0]), dy = __fsub_rn(M[t * 6 + 1], s[1]);
                const float dz = __fsub_rn(M[t * 6 + 2], s[2]);
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
        const float* tm = M + (size_t)t * 6;
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

}  // namespace

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
  if (!frame_idx || !rendered_depth || !boxes || !T0 || !K || !out_poses || !out_status || !out_residual ||
      !out_fitness || !workspace)
    return fail(GP_ERR_INVALID, "null argument");
  if (p.debug.trace && (p.debug.trace_capacity < 1 || !p.debug.trace_count))
    return fail(GP_ERR_INVALID, "debug.trace needs trace_capacity >= 1 and trace_count");
  if (n_hyp == 0) return GP_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const size_t plane = (size_t)height * width;
  char* ws = static_cast<char*>(workspace);
  const float* map = reinterpret_cast<const float*>(ws);
  int* src = reinterpret_cast<int*>(ws + scene_bytes(n_frames, height, width));
  unsigned* dist = reinterpret_cast<unsigned*>(src + n_hyp * plane);
  int* tgt = reinterpret_cast<int*>(dist + n_hyp * plane);
  GP_CUDA(gp::launch_ex(icp_kernel, n_hyp, kThreads, 0, st, 1, false, n_frames, height, width, frame_idx, masks,
                        rendered_depth, boxes, T0, K, map, p, src, dist, tgt, out_poses, out_status, out_residual,
                        out_fitness));
  return GP_OK;
}

extern "C" int gp_debug_icp_select(const uint32_t* bits, int n, int rank, uint32_t* out, void* stream) {
  if (n < 1) return fail(GP_ERR_INVALID, "n %d must be >= 1", n);
  if (rank < 0 || rank >= n) return fail(GP_ERR_INVALID, "rank %d outside [0, n = %d)", rank, n);
  if (!bits || !out) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(select_kernel, 1, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false, bits, n, rank, out));
  return GP_OK;
}
