// Row f7: the BOP 2019 pose-error metrics on the GPU, in place of the external BOP toolkit's eval_bop19_pose.py that
// the reference calls (src/scripts/eval_bop.py:16-38).  Definitions: VSD, Hodan et al., "BOP: Benchmark for 6D Object
// Pose Estimation", ECCV 2018; MSSD and MSPD, Hodan et al., "BOP Challenge 2020 on 6D Object Localization".
// The host side (gigapose_b200/bop_eval.py) pairs estimates with ground truths, renders both with gp_render_depth and
// matches the errors into recalls.
//
// Contract (what tests/test_gpu_bop_eval.py pins against oracle/bop_port.py, bit for bit):
//  gp_bop_vsd, one CTA per (estimate, ground truth) pair, walking the union of the two render boxes (clipped to the
//  image; no other pixel can be in either visibility mask).  Every operation below is one fp32 rounding
//  (__fmul_rn / __fadd_rn / __fsub_rn / __fdiv_rn / __fsqrt_rn), no FMA contraction:
//    distance of a depth z at pixel (u, v), K = [fx . cx; . fy cy] of the pair's frame (the skew is not used):
//      X = ((u - cx) * z) / fx,  Y = ((v - cy) * z) / fy,  dist = sqrt((X * X + Y * Y) + z * z)   (0 for z = 0)
//    with u, v the integer column and row (the rasteriser's pixel centre), for the test, estimate and GT depths;
//    visib_gt  = dist_gt > 0 and ((dist_gt - dist_test) <= delta or dist_test == 0)
//    visib_est = (dist_est > 0 and ((dist_est - dist_test) <= delta or dist_test == 0)) or (visib_gt and dist_est > 0)
//    inter / union = pixels in both / either mask;  cost_t = pixels of inter with
//      |dist_gt - dist_est| / diameter >= tau_t
//    counts [n, 2 + n_tau] i32 = (inter, union, cost_0, ...);  e_t = float(cost_t + union - inter) / float(union),
//    1 when union = 0 (an integer sum, then one rounding each to fp32, then one division).
//  gp_bop_mssd_mspd, one CTA per (pair, chunk of kSymPerCta symmetry transforms) of the pair's object, threads over its
//  vertices x:  s = S x (S = [S_R | S_t] of the transform),  g = P_gt s,  e = P_est x, each row ((A0 x + A1 y) + A2 z)
//  + A3;  MSSD term = (dx * dx + dy * dy) + dz * dz with d = e - g;  MSPD term the same over the pixel differences of
//  the two projections u = (K00 x + K01 y) / z + K02, v = (K11 y) / z + K12 (the rasteriser's projection).  The max
//  over vertices is taken on the squared terms, then one sqrt, then the min over transforms with an atomicMin on the
//  float bits: every value is >= 0 or NaN, so the unsigned bit order is the float order with NaN last, and both the
//  max and the min are exact and independent of the schedule.
//
// Row f8: the BOP 2024 6D-detection score (the toolkit's eval_bop24_pose.py that the reference's README points to for
// `test_setting: detection` runs), with COCO's rules for ranking, ignored ground truths and interpolated precision
// (Lin et al., "Microsoft COCO: Common Objects in Context", ECCV 2014).  This is this repository's statement of it; it is
// unverified against eval_bop24_pose.py.  The host side (gigapose_b200/bop_eval.py, prepare_detection) keeps the
// max_estimates_per_image highest-scoring estimates of each target image (stable: csv order on ties), calls a ground
// truth valid when its visib_fract >= 0.1 and ignored otherwise, evaluates the objects with at least one valid ground
// truth, and computes MSSD / MSPD of every (kept estimate, ground truth of its object in its image) pair with
// gp_bop_mssd_mspd.  Thresholds are fp64 (theta x diameter, theta x width / 640), computed on the host.
//  gp_bop_match, one warp per (group = (image, object), metric, threshold): the group's estimates in descending score
//  order (csv order on ties), each in turn:
//    1. takes the unmatched valid ground truth with the smallest double(err) < thr (the lowest index on a tie): TP;
//    2. else takes the unmatched ignored ground truth with the smallest double(err) < thr (lowest index): ignored;
//    3. else FP.
//  A NaN error fails `<` and never matches.  Lane l owns the ground truths j = 32 c + l and keeps their taken flags as
//  bit c of one register (hence at most 32 x 32 ground truths per group); the arg-min is a butterfly on (error, index).
//  gp_bop_average_precision, one CTA per (object, metric, threshold) over the object's estimates ranked by score over
//  all images (a host stable argsort): inclusive integer block scans of TP and FP (ignored estimates keep their rank and
//  add to neither), then per rank, in fp64, recall = TP / n_valid and precision = TP / ((TP + FP) + 2^-52), each one
//  IEEE operation (__ddiv_rn / __dadd_rn).  The COCO interpolation q_k = max { precision_j : j >= first rank with
//  recall >= r_k } (0 when no rank reaches r_k) equals max { precision_j : recall_j >= r_k } because the recall is
//  non-decreasing, so each rank binary-searches c_j = #{k : r_k <= recall_j} and takes an atomicMax of its precision
//  bits into slot c_j (precisions are >= 0, so the unsigned bit order is the double order and the max is exact); a
//  suffix max over the slots gives q_k = max over slots c > k.  AP = (((q_0 + q_1) + q_2) + ... + q_{K-1}) / K in fp64,
//  summed on one thread.  Every step is an integer operation, an exact max or one rounded fp64 operation, so
//  oracle/bop24_port.py (detection_labels, average_precision) restates it bit for bit.
//
// Row f12: ADD, ADD-S and the 2D-projection error (gp_bop_add); the definitions are the comment above add_kernel.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

#include <cstring>
#include <vector>

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kSymPerCta = 8;

struct Taus {
  float v[GP_BOP_MAX_TAU];
};

struct ObjectTables {                 // host offsets, by value: object o owns [off[o], off[o + 1])
  int32_t vert_off[GP_BOP_MAX_OBJECTS + 1];
  int32_t sym_off[GP_BOP_MAX_OBJECTS + 1];
};

__device__ __forceinline__ float distance(float z, int u, int v, float fx, float fy, float cx, float cy) {
  const float X = __fdiv_rn(__fmul_rn(__fsub_rn((float)u, cx), z), fx);
  const float Y = __fdiv_rn(__fmul_rn(__fsub_rn((float)v, cy), z), fy);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(X, X), __fmul_rn(Y, Y)), __fmul_rn(z, z)));
}

__device__ __forceinline__ bool visible(float d_model, float d_test, float delta) {
  return d_model > 0.f && (__fsub_rn(d_model, d_test) <= delta || d_test == 0.f);
}

__global__ void __launch_bounds__(kThreads)
vsd_kernel(int n_frames, int H, int W, const float* __restrict__ depth_test, const float* __restrict__ Kmat,
           const int32_t* __restrict__ frame_idx, int n_est, const float* __restrict__ est_depth,
           const long long* __restrict__ est_boxes, const int32_t* __restrict__ est_idx, int n_gt,
           const float* __restrict__ gt_depth, const long long* __restrict__ gt_boxes,
           const int32_t* __restrict__ gt_idx, const float* __restrict__ diameter, float delta, int n_tau, Taus taus,
           int32_t* __restrict__ counts, float* __restrict__ errors) {
  __shared__ int red[kWarps][2 + GP_BOP_MAX_TAU];
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f = frame_idx[pair], ie = est_idx[pair], ig = gt_idx[pair];
  const int ncol = 2 + n_tau;
  if (f < 0 || f >= n_frames || ie < 0 || ie >= n_est || ig < 0 || ig >= n_gt) {
    for (int c = tid; c < ncol; c += kThreads) counts[(size_t)pair * ncol + c] = -1;
    for (int c = tid; c < n_tau; c += kThreads) errors[(size_t)pair * n_tau + c] = __int_as_float(0x7fffffff);
    return;
  }
  const float* K = Kmat + 9 * (size_t)f;
  const float fx = K[0], cx = K[2], fy = K[4], cy = K[5];
  const float diam = diameter[pair];
  const long long* be = est_boxes + 4 * (size_t)ie;
  const long long* bg = gt_boxes + 4 * (size_t)ig;
  const int x0 = (int)max(min(be[0], bg[0]), 0ll), y0 = (int)max(min(be[1], bg[1]), 0ll);
  const int x1 = (int)min(max(be[2], bg[2]), (long long)W), y1 = (int)min(max(be[3], bg[3]), (long long)H);
  const size_t plane = (size_t)H * W;
  const float* dt = depth_test + f * plane;
  const float* de = est_depth + ie * plane;
  const float* dg = gt_depth + ig * plane;
  int cnt[2 + GP_BOP_MAX_TAU];
#pragma unroll
  for (int c = 0; c < 2 + GP_BOP_MAX_TAU; ++c) cnt[c] = 0;
  const int bw = max(x1 - x0, 0), n = bw * max(y1 - y0, 0);
  for (int p = tid; p < n; p += kThreads) {
    const int v = y0 + p / bw, u = x0 + p % bw;
    const size_t i = (size_t)v * W + u;
    const float d_test = distance(dt[i], u, v, fx, fy, cx, cy);
    const float d_gt = distance(dg[i], u, v, fx, fy, cx, cy);
    const float d_est = distance(de[i], u, v, fx, fy, cx, cy);
    const bool vg = visible(d_gt, d_test, delta);
    const bool ve = visible(d_est, d_test, delta) || (vg && d_est > 0.f);
    if (vg && ve) {
      ++cnt[0];
      const float c = __fdiv_rn(fabsf(__fsub_rn(d_gt, d_est)), diam);
#pragma unroll
      for (int t = 0; t < GP_BOP_MAX_TAU; ++t)
        if (t < n_tau && c >= taus.v[t]) ++cnt[2 + t];
    }
    if (vg || ve) ++cnt[1];
  }
#pragma unroll
  for (int c = 0; c < 2 + GP_BOP_MAX_TAU; ++c) {
    const int s = __reduce_add_sync(0xffffffffu, cnt[c]);
    if (lane == 0 && c < ncol) red[warp][c] = s;
  }
  __syncthreads();
  if (tid < ncol) {
    int s = 0;
    for (int w = 0; w < kWarps; ++w) s += red[w][tid];
    counts[(size_t)pair * ncol + tid] = s;
    red[0][tid] = s;                    // column tid is read by no other thread before the barrier
  }
  __syncthreads();
  if (tid < n_tau) {
    const int inter = red[0][0], uni = red[0][1];
    errors[(size_t)pair * n_tau + tid] =
        uni == 0 ? 1.f : __fdiv_rn((float)(red[0][2 + tid] + uni - inter), (float)uni);
  }
}

// ((A0 x + A1 y) + A2 z) + A3 for the three rows of a row-major [3,4] (or the top of a [4,4]) matrix
__device__ __forceinline__ void affine(const float* A, float x, float y, float z, float o[3]) {
#pragma unroll
  for (int r = 0; r < 3; ++r)
    o[r] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(A[4 * r], x), __fmul_rn(A[4 * r + 1], y)), __fmul_rn(A[4 * r + 2], z)),
                     A[4 * r + 3]);
}

__device__ __forceinline__ void project(const float* K, const float p[3], float& u, float& v) {
  u = __fadd_rn(__fdiv_rn(__fadd_rn(__fmul_rn(K[0], p[0]), __fmul_rn(K[1], p[1])), p[2]), K[2]);
  v = __fadd_rn(__fdiv_rn(__fmul_rn(K[4], p[1]), p[2]), K[5]);
}

__device__ __forceinline__ float sq3(float a, float b, float c) {
  return __fadd_rn(__fadd_rn(__fmul_rn(a, a), __fmul_rn(b, b)), __fmul_rn(c, c));
}

__global__ void __launch_bounds__(kThreads)
mssd_mspd_kernel(int n_objects, const int32_t* __restrict__ obj_idx, ObjectTables tab, const float* __restrict__ vertices,
                 const float* __restrict__ syms, int n_frames, const float* __restrict__ Kmat,
                 const int32_t* __restrict__ frame_idx, const float* __restrict__ pose_est,
                 const float* __restrict__ pose_gt, float* __restrict__ mssd, float* __restrict__ mspd) {
  __shared__ float sS[kSymPerCta][16], sPe[16], sPg[16], sK[9];
  __shared__ unsigned red[kWarps][2 * kSymPerCta];
  const int pair = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int o = obj_idx[pair], f = frame_idx[pair];
  if (o < 0 || o >= n_objects || f < 0 || f >= n_frames) return;    // outputs keep their all-ones (NaN) bits
  const int s0 = tab.sym_off[o] + blockIdx.y * kSymPerCta;
  const int ns = min(tab.sym_off[o + 1] - s0, kSymPerCta);
  if (ns <= 0) return;
  for (int i = tid; i < ns * 16; i += kThreads) sS[i / 16][i % 16] = syms[16 * (size_t)s0 + i];
  if (tid < 16) { sPe[tid] = pose_est[16 * (size_t)pair + tid]; sPg[tid] = pose_gt[16 * (size_t)pair + tid]; }
  if (tid < 9) sK[tid] = Kmat[9 * (size_t)f + tid];
  __syncthreads();
  unsigned md[kSymPerCta], mp[kSymPerCta];
#pragma unroll
  for (int s = 0; s < kSymPerCta; ++s) md[s] = mp[s] = 0u;
  const int v0 = tab.vert_off[o], v1 = tab.vert_off[o + 1];
  for (int i = v0 + tid; i < v1; i += kThreads) {
    const float x = vertices[3 * (size_t)i], y = vertices[3 * (size_t)i + 1], z = vertices[3 * (size_t)i + 2];
    float e[3], ue, ve;
    affine(sPe, x, y, z, e);
    project(sK, e, ue, ve);
#pragma unroll
    for (int s = 0; s < kSymPerCta; ++s) {
      if (s >= ns) break;
      float sx[3], g[3], ug, vg;
      affine(sS[s], x, y, z, sx);
      affine(sPg, sx[0], sx[1], sx[2], g);
      project(sK, g, ug, vg);
      const float d = sq3(__fsub_rn(e[0], g[0]), __fsub_rn(e[1], g[1]), __fsub_rn(e[2], g[2]));
      const float du = __fsub_rn(ue, ug), dv = __fsub_rn(ve, vg);
      const float p = __fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv));
      md[s] = max(md[s], __float_as_uint(d));
      mp[s] = max(mp[s], __float_as_uint(p));
    }
  }
#pragma unroll
  for (int s = 0; s < kSymPerCta; ++s) {
    const unsigned a = __reduce_max_sync(0xffffffffu, md[s]), b = __reduce_max_sync(0xffffffffu, mp[s]);
    if (lane == 0) { red[warp][s] = a; red[warp][kSymPerCta + s] = b; }
  }
  __syncthreads();
  if (tid < 2) {
    unsigned best = 0xffffffffu;
    for (int s = 0; s < ns; ++s) {
      unsigned m = 0u;
      for (int w = 0; w < kWarps; ++w) m = max(m, red[w][tid * kSymPerCta + s]);
      best = min(best, __float_as_uint(__fsqrt_rn(__uint_as_float(m))));
    }
    atomicMin(reinterpret_cast<unsigned*>(tid == 0 ? mssd : mspd) + pair, best);
  }
}

constexpr int kMaxSide = 8192;

// ---------------------------------------------------------------------------------------------------- row f8
struct MatchGroup {                   // GP_BOP_MATCH_GROUP_BYTES; gp_bop_match copies one per group into its workspace
  long long err0;                     // first error of the group's dense [n_est, n_gt] block
  int32_t est0, n_est, gt0, n_gt, obj, pad;
};
static_assert(sizeof(MatchGroup) == GP_BOP_MATCH_GROUP_BYTES, "MatchGroup layout");

// arg-min over the warp of (d, j), the lower j on equal d; every lane ends with the same pair
__device__ __forceinline__ void warp_argmin(double& d, int& j) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const double d2 = __shfl_xor_sync(0xffffffffu, d, o);
    const int j2 = __shfl_xor_sync(0xffffffffu, j, o);
    if (d2 < d || (d2 == d && j2 < j)) { d = d2; j = j2; }
  }
}

constexpr int kNone = 0x7fffffff;

__global__ void __launch_bounds__(kThreads)
match_kernel(long long n_warps, int n_theta, const MatchGroup* __restrict__ groups, const double* __restrict__ thr,
             const float* __restrict__ mssd, const float* __restrict__ mspd, const uint8_t* __restrict__ gt_valid,
             int8_t* __restrict__ labels) {
  const long long w = ((long long)blockIdx.x * kThreads + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= n_warps) return;                                  // whole warps: kThreads is a multiple of 32
  const int g = (int)(w / (2 * n_theta)), m = (int)(w / n_theta) & 1, t = (int)(w % n_theta);
  const MatchGroup G = groups[g];
  const double th = thr[((size_t)G.obj * 2 + m) * n_theta + t];
  const float* err = (m == 0 ? mssd : mspd) + G.err0;
  const int chunks = (G.n_gt + 31) >> 5;
  unsigned valid = 0u, taken = 0u;                           // bit c: ground truth 32 c + lane
  for (int c = 0; c < chunks; ++c) {
    const int j = 32 * c + lane;
    if (j < G.n_gt && gt_valid[G.gt0 + j]) valid |= 1u << c;
  }
  for (int a = 0; a < G.n_est; ++a) {
    const float* row = err + (long long)a * G.n_gt;
    double dv = __longlong_as_double(0x7ff0000000000000ll), di = dv;
    int jv = kNone, ji = kNone;
    for (int c = 0; c < chunks; ++c) {                       // ascending j per lane: strict < keeps the lowest
      const int j = 32 * c + lane;
      if (j >= G.n_gt || ((taken >> c) & 1u)) continue;
      const double d = (double)row[j];
      if (!(d < th)) continue;
      if ((valid >> c) & 1u) {
        if (d < dv) { dv = d; jv = j; }
      } else if (d < di) {
        di = d;
        ji = j;
      }
    }
    warp_argmin(dv, jv);
    int label = GP_BOP_LABEL_FP, take = kNone;
    if (jv != kNone) {
      label = GP_BOP_LABEL_TP;
      take = jv;
    } else {
      warp_argmin(di, ji);                                   // warp-uniform branch: jv is the same on every lane
      if (ji != kNone) { label = GP_BOP_LABEL_IGNORED; take = ji; }
    }
    if (take != kNone && (take & 31) == lane) taken |= 1u << (take >> 5);
    if (lane == 0) labels[((size_t)(G.est0 + a) * 2 + m) * n_theta + t] = (int8_t)label;
  }
}

struct ApTables {                     // host tables, by value: object o ranks rank[off[o] .. off[o + 1])
  int32_t rank_off[GP_BOP_MAX_OBJECTS + 1];
  int32_t n_valid[GP_BOP_MAX_OBJECTS];
  double recall[GP_BOP_MAX_RECALL];
};

__global__ void __launch_bounds__(kThreads)
ap_kernel(int n_theta, int n_est, const int8_t* __restrict__ labels, const int32_t* __restrict__ rank, int n_recall,
          ApTables tab, double* __restrict__ ap) {
  __shared__ unsigned long long best[GP_BOP_MAX_RECALL + 1];  // slot c: max precision bits of ranks with c_j = c
  __shared__ double rthr[GP_BOP_MAX_RECALL];
  __shared__ int wsum[2][kWarps];
  __shared__ int bad;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int o = blockIdx.x / (2 * n_theta), m = (blockIdx.x / n_theta) & 1, t = blockIdx.x % n_theta;
  for (int c = tid; c <= n_recall; c += kThreads) best[c] = 0ull;
  for (int c = tid; c < n_recall; c += kThreads) rthr[c] = tab.recall[c];
  if (tid == 0) bad = 0;
  __syncthreads();
  const int r0 = tab.rank_off[o], n = tab.rank_off[o + 1] - r0;
  const double nv = (double)tab.n_valid[o];
  int carry_tp = 0, carry_fp = 0;
  for (int base = 0; base < n; base += kThreads) {
    const int i = base + tid;
    int tp = 0, fp = 0;
    if (i < n) {
      const int e = rank[r0 + i];
      if (e < 0 || e >= n_est) {
        bad = 1;
      } else {
        const int L = labels[((size_t)e * 2 + m) * n_theta + t];
        tp = L == GP_BOP_LABEL_TP;
        fp = L == GP_BOP_LABEL_FP;
      }
    }
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {                       // inclusive warp scans
      const int a = __shfl_up_sync(0xffffffffu, tp, d), b = __shfl_up_sync(0xffffffffu, fp, d);
      if (lane >= d) { tp += a; fp += b; }
    }
    if (lane == 31) { wsum[0][warp] = tp; wsum[1][warp] = fp; }
    __syncthreads();
    int tile_tp = 0, tile_fp = 0;
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      if (w < warp) { tp += wsum[0][w]; fp += wsum[1][w]; }
      tile_tp += wsum[0][w];
      tile_fp += wsum[1][w];
    }
    __syncthreads();                                         // wsum is rewritten by the next tile
    if (i < n) {
      const int TP = carry_tp + tp, FP = carry_fp + fp;
      const double rc = __ddiv_rn((double)TP, nv);
      const double pr = __ddiv_rn((double)TP, __dadd_rn((double)(TP + FP), 0x1p-52));
      int lo = 0, hi = n_recall;                             // c_j = #{k : r_k <= recall_j}
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (rthr[mid] <= rc) lo = mid + 1; else hi = mid;
      }
      if (lo > 0) atomicMax(&best[lo], (unsigned long long)__double_as_longlong(pr));
    }
    carry_tp += tile_tp;
    carry_fp += tile_fp;
  }
  __syncthreads();
  if (tid == 0) {
    for (int c = n_recall - 1; c >= 1; --c) best[c] = max(best[c], best[c + 1]);
    double sum = 0.0;
    for (int k = 0; k < n_recall; ++k) sum = __dadd_rn(sum, __longlong_as_double((long long)best[k + 1]));
    ap[blockIdx.x] = bad ? __longlong_as_double(0x7ff8000000000000ll) : __ddiv_rn(sum, (double)n_recall);
  }
}

// ---------------------------------------------------------------------------------------------------- row f12
// ADD (Hinterstoisser et al., ACCV 2012), ADD-S (the same paper's measure for indistinguishable views; PoseCNN's "ADD-S")
// and the 2D-projection error (Brachmann et al., CVPR 2016) of (estimate, ground truth) pairs of the same object.  P =
// [R | t] object -> camera; the model points x are all vertices of the object (N of them), in the model unit.
//   ADD   = mean over x of |P_est x - P_gt x|
//   ADD-S = mean over the ground-truth points g_j = P_gt x_j of min over i of |g_j - P_est x_i|   (the nearest
//           estimated point of each ground-truth point: the direction of MegaPose's dists_add_symmetric and of the BOP
//           toolkit's adi)
//   proj  = mean over x of the pixel distance between the projections of P_est x and P_gt x with the frame's K
// Per-vertex arithmetic is mssd_mspd_kernel's with S = I: e = P_est x and g = P_gt x by `affine`, each row
// ((A0 x + A1 y) + A2 z) + A3; squared distance `sq3` = (dx dx + dy dy) + dz dz with d = e - g; projection `project`,
// u = (K00 x + K01 y) / z + K02, v = (K11 y) / z + K12, squared pixel distance du du + dv dv; every operation one fp32
// rounding, no FMA contraction.  The per-point distances are one __fsqrt_rn of the squared term; for ADD-S the min over
// i is taken on the squared terms first (as unsigned bits: every term is >= 0 or NaN, so it is the float order with NaN
// above +inf; a NaN term wins only when every term is NaN), then one sqrt.  The min is exact, so the schedule does not
// matter.
// Sums: vertex j belongs to chunk c = j / GP_BOP_ADD_CHUNK.  Each chunk's partial is the fp64 sum of its per-point
// distances widened to fp64, left to right in vertex order, starting from the first; the finishing launch adds the
// partials left to right in chunk order and divides once by (double)N (__ddiv_rn).  Nothing else enters the order, so
// oracle/add_port.py restates it bit for bit.  A pair whose object or frame index is out of range gets NaN; a NaN pose
// gives NaN.
// Schedule: grid (pair, chunk), kThreads threads, thread t holding the ground-truth vertices c * CHUNK + t + kThreads r
// (r < kAddPerThread) in registers with their ADD and proj terms; the estimated points of the object are transformed into
// shared-memory tiles of kAddTile points and streamed past them.  The partials go to the workspace
// (f64 [n_pairs, n_chunks, 3]); add_finish_kernel sums them, one thread per (pair, metric).
constexpr int kAddPerThread = GP_BOP_ADD_CHUNK / kThreads;
constexpr int kAddTile = 1024;
static_assert(kAddPerThread * kThreads == GP_BOP_ADD_CHUNK, "chunk = threads x vertices per thread");

struct VertexTable {                  // host offsets, by value: object o owns vertices [off[o], off[o + 1])
  int32_t off[GP_BOP_MAX_OBJECTS + 1];
};

// Row f14 (gp_vis_vertex_errors, csrc/vis.cu) runs the same kernel with kPerVertex = true: no projection, and instead of
// the chunk partials it stores each ground-truth vertex's ADD distance (symmetric[pair] = 0) or ADD-S distance (!= 0)
// at values[out_off[pair] + j].  A pair whose object index is out of range, or whose slot out_off[pair + 1] -
// out_off[pair] is not the object's vertex count, gets NaN over the part of its slot that the grid covers.
template <bool kPerVertex>
__global__ void __launch_bounds__(kThreads, 2)
add_kernel(int n_objects, const int32_t* __restrict__ obj_idx, VertexTable tab, const float* __restrict__ vertices,
           int n_frames, const float* __restrict__ Kmat, const int32_t* __restrict__ frame_idx,
           const float* __restrict__ pose_est, const float* __restrict__ pose_gt, double* __restrict__ partial,
           const uint8_t* __restrict__ symmetric, const long long* __restrict__ out_off, float* __restrict__ values) {
  __shared__ float4 sE[kAddTile];
  __shared__ float sDist[3][kPerVertex ? 1 : GP_BOP_ADD_CHUNK];
  __shared__ float sPe[16], sPg[16], sK[9];
  const int pair = blockIdx.x, chunk = blockIdx.y, tid = threadIdx.x;
  const int o = obj_idx[pair], f = kPerVertex ? 0 : frame_idx[pair];
  const int j0 = chunk * GP_BOP_ADD_CHUNK;
  if constexpr (kPerVertex) {
    const long long s0 = out_off[pair], len = out_off[pair + 1] - s0;
    if (o < 0 || o >= n_objects || len != tab.off[o + 1] - tab.off[o]) {
      for (int r = 0; r < kAddPerThread; ++r) {
        const long long j = j0 + tid + kThreads * r;
        if (j < len) values[s0 + j] = __int_as_float(0x7fffffff);
      }
      return;
    }
  } else if (o < 0 || o >= n_objects || f < 0 || f >= n_frames) {
    return;                                                  // add_finish_kernel writes NaN
  }
  const int v0 = tab.off[o], n = tab.off[o + 1] - v0;
  if (j0 >= n) return;
  const bool min_needed = !kPerVertex || symmetric[pair];
  if (tid < 16) { sPe[tid] = pose_est[16 * (size_t)pair + tid]; sPg[tid] = pose_gt[16 * (size_t)pair + tid]; }
  if (!kPerVertex && tid < 9) sK[tid] = Kmat[9 * (size_t)f + tid];
  __syncthreads();
  float g[kAddPerThread][3];
  float add[kAddPerThread];
  unsigned best[kAddPerThread];
#pragma unroll
  for (int r = 0; r < kAddPerThread; ++r) {
    const int j = j0 + tid + kThreads * r;
    best[r] = 0xffffffffu;
    if (j < n) {
      const float* p = vertices + 3 * (size_t)(v0 + j);
      const float x = p[0], y = p[1], z = p[2];
      float e[3];
      affine(sPe, x, y, z, e);
      affine(sPg, x, y, z, g[r]);
      add[r] = __fsqrt_rn(sq3(__fsub_rn(e[0], g[r][0]), __fsub_rn(e[1], g[r][1]), __fsub_rn(e[2], g[r][2])));
      if constexpr (!kPerVertex) {
        float ue, ve, ug, vg;
        project(sK, e, ue, ve);
        project(sK, g[r], ug, vg);
        const float du = __fsub_rn(ue, ug), dv = __fsub_rn(ve, vg);
        sDist[0][tid + kThreads * r] = add[r];
        sDist[2][tid + kThreads * r] = __fsqrt_rn(__fadd_rn(__fmul_rn(du, du), __fmul_rn(dv, dv)));
      }
    } else {
      g[r][0] = g[r][1] = g[r][2] = 0.f;
      add[r] = 0.f;
    }
  }
  for (int base = 0; min_needed && base < n; base += kAddTile) {   // min_needed is uniform over the CTA
    const int m = min(kAddTile, n - base);
    __syncthreads();                                         // the previous tile has been read
    for (int i = tid; i < m; i += kThreads) {
      const float* p = vertices + 3 * (size_t)(v0 + base + i);
      float e[3];
      affine(sPe, p[0], p[1], p[2], e);
      sE[i] = make_float4(e[0], e[1], e[2], 0.f);
    }
    __syncthreads();
#pragma unroll 4
    for (int i = 0; i < m; ++i) {
      const float4 e = sE[i];                                // the same address on every lane: a broadcast
#pragma unroll
      for (int r = 0; r < kAddPerThread; ++r)
        best[r] = min(best[r], __float_as_uint(sq3(__fsub_rn(e.x, g[r][0]), __fsub_rn(e.y, g[r][1]),
                                                   __fsub_rn(e.z, g[r][2]))));
    }
  }
  if constexpr (kPerVertex) {
    const long long s0 = out_off[pair];
#pragma unroll
    for (int r = 0; r < kAddPerThread; ++r) {
      const int j = j0 + tid + kThreads * r;
      if (j < n) values[s0 + j] = min_needed ? __fsqrt_rn(__uint_as_float(best[r])) : add[r];
    }
  } else {
#pragma unroll
    for (int r = 0; r < kAddPerThread; ++r)
      if (j0 + tid + kThreads * r < n) sDist[1][tid + kThreads * r] = __fsqrt_rn(__uint_as_float(best[r]));
    __syncthreads();
    if (tid < 3) {
      const int cnt = min(GP_BOP_ADD_CHUNK, n - j0);
      double s = (double)sDist[tid][0];
      for (int j = 1; j < cnt; ++j) s = __dadd_rn(s, (double)sDist[tid][j]);
      partial[((size_t)pair * gridDim.y + chunk) * 3 + tid] = s;
    }
  }
}

__global__ void __launch_bounds__(kThreads)
add_finish_kernel(int n_pairs, int n_chunks, int n_objects, const int32_t* __restrict__ obj_idx, VertexTable tab,
                  int n_frames, const int32_t* __restrict__ frame_idx, const double* __restrict__ partial,
                  double* __restrict__ out) {
  const long long t = (long long)blockIdx.x * kThreads + threadIdx.x;
  if (t >= 3ll * n_pairs) return;
  const int pair = (int)(t / 3), m = (int)(t % 3);
  const int o = obj_idx[pair], f = frame_idx[pair];
  if (o < 0 || o >= n_objects || f < 0 || f >= n_frames) {
    out[t] = __longlong_as_double(0x7ff8000000000000ll);
    return;
  }
  const int n = tab.off[o + 1] - tab.off[o];
  const int nc = (n + GP_BOP_ADD_CHUNK - 1) / GP_BOP_ADD_CHUNK;
  const double* p = partial + (size_t)pair * n_chunks * 3 + m;
  double s = p[0];
  for (int c = 1; c < nc; ++c) s = __dadd_rn(s, p[3 * c]);
  out[t] = __ddiv_rn(s, (double)n);
}

}  // namespace

extern "C" int gp_bop_vsd(int n_pairs, int n_frames, int height, int width, const float* depth_test, const float* K,
                          const int32_t* frame_idx, int n_est, const float* est_depth, const int64_t* est_boxes,
                          const int32_t* est_idx, int n_gt, const float* gt_depth, const int64_t* gt_boxes,
                          const int32_t* gt_idx, const float* diameter, float delta, int n_tau, const float* tau,
                          int32_t* counts, float* errors, void* stream) {
  if (n_pairs < 1) return fail(GP_ERR_INVALID, "n_pairs %d must be >= 1", n_pairs);
  if (n_frames < 1 || n_est < 1 || n_gt < 1)
    return fail(GP_ERR_INVALID, "n_frames %d, n_est %d, n_gt %d must be >= 1", n_frames, n_est, n_gt);
  if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [1, %d]", height, width, kMaxSide);
  if (n_tau < 1 || n_tau > GP_BOP_MAX_TAU) return fail(GP_ERR_INVALID, "n_tau %d outside [1, %d]", n_tau, GP_BOP_MAX_TAU);
  if (!(delta > 0.f) || !isfinite(delta)) return fail(GP_ERR_INVALID, "delta must be positive and finite");
  if (!tau) return fail(GP_ERR_INVALID, "null tau");
  Taus taus;
  for (int t = 0; t < n_tau; ++t) {
    if (!(tau[t] > 0.f) || !isfinite(tau[t])) return fail(GP_ERR_INVALID, "tau[%d] must be positive and finite", t);
    taus.v[t] = tau[t];
  }
  for (int t = n_tau; t < GP_BOP_MAX_TAU; ++t) taus.v[t] = 0.f;
  if (!depth_test || !K || !frame_idx || !est_depth || !est_boxes || !est_idx || !gt_depth || !gt_boxes || !gt_idx ||
      !diameter || !counts || !errors)
    return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(vsd_kernel, n_pairs, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false, n_frames, height,
                        width, depth_test, K, frame_idx, n_est, est_depth, reinterpret_cast<const long long*>(est_boxes),
                        est_idx, n_gt, gt_depth, reinterpret_cast<const long long*>(gt_boxes), gt_idx, diameter, delta,
                        n_tau, taus, counts, errors));
  return GP_OK;
}

extern "C" int gp_bop_mssd_mspd(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets,
                                const float* vertices, const int32_t* sym_offsets, const float* syms, int n_frames,
                                const float* K, const int32_t* frame_idx, const float* pose_est, const float* pose_gt,
                                float* mssd, float* mspd, void* stream) {
  if (n_pairs < 1) return fail(GP_ERR_INVALID, "n_pairs %d must be >= 1", n_pairs);
  if (n_objects < 1 || n_objects > GP_BOP_MAX_OBJECTS)
    return fail(GP_ERR_INVALID, "n_objects %d outside [1, %d]", n_objects, GP_BOP_MAX_OBJECTS);
  if (n_frames < 1) return fail(GP_ERR_INVALID, "n_frames %d must be >= 1", n_frames);
  if (!vertex_offsets || !sym_offsets) return fail(GP_ERR_INVALID, "null offsets");
  ObjectTables tab;
  int max_syms = 0;
  for (int o = 0; o <= n_objects; ++o) {
    tab.vert_off[o] = vertex_offsets[o];
    tab.sym_off[o] = sym_offsets[o];
    if (o == 0 ? vertex_offsets[0] != 0 || sym_offsets[0] != 0
               : vertex_offsets[o] <= vertex_offsets[o - 1] || sym_offsets[o] <= sym_offsets[o - 1])
      return fail(GP_ERR_INVALID, "bad offsets at object %d: they must start at 0 and increase strictly "
                  "(every object has a vertex and a transform)", o);
    if (o > 0) max_syms = max(max_syms, sym_offsets[o] - sym_offsets[o - 1]);
  }
  for (int o = n_objects + 1; o <= GP_BOP_MAX_OBJECTS; ++o) tab.vert_off[o] = tab.sym_off[o] = 0;
  if (!obj_idx || !vertices || !syms || !K || !frame_idx || !pose_est || !pose_gt || !mssd || !mspd)
    return fail(GP_ERR_INVALID, "null argument");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GP_CUDA(cudaMemsetAsync(mssd, 0xFF, (size_t)n_pairs * sizeof(float), st));
  GP_CUDA(cudaMemsetAsync(mspd, 0xFF, (size_t)n_pairs * sizeof(float), st));
  GP_CUDA(gp::launch_ex(mssd_mspd_kernel, dim3(n_pairs, (max_syms + kSymPerCta - 1) / kSymPerCta), kThreads, 0, st, 1,
                        false, n_objects, obj_idx, tab, vertices, syms, n_frames, K, frame_idx, pose_est, pose_gt, mssd,
                        mspd));
  return GP_OK;
}

extern "C" int gp_bop_add(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets,
                          const float* vertices, int n_frames, const float* K, const int32_t* frame_idx,
                          const float* pose_est, const float* pose_gt, void* workspace, double* out, void* stream) {
  if (n_pairs < 1) return fail(GP_ERR_INVALID, "n_pairs %d must be >= 1", n_pairs);
  if (n_objects < 1 || n_objects > GP_BOP_MAX_OBJECTS)
    return fail(GP_ERR_INVALID, "n_objects %d outside [1, %d]", n_objects, GP_BOP_MAX_OBJECTS);
  if (n_frames < 1) return fail(GP_ERR_INVALID, "n_frames %d must be >= 1", n_frames);
  if (!vertex_offsets) return fail(GP_ERR_INVALID, "null offsets");
  VertexTable tab;
  int max_v = 0;
  for (int o = 0; o <= n_objects; ++o) {
    tab.off[o] = vertex_offsets[o];
    if (o == 0 ? vertex_offsets[0] != 0 : vertex_offsets[o] <= vertex_offsets[o - 1])
      return fail(GP_ERR_INVALID, "bad vertex offsets at object %d: they must start at 0 and increase strictly", o);
    if (o > 0) max_v = max(max_v, vertex_offsets[o] - vertex_offsets[o - 1]);
  }
  for (int o = n_objects + 1; o <= GP_BOP_MAX_OBJECTS; ++o) tab.off[o] = 0;
  const int n_chunks = (max_v + GP_BOP_ADD_CHUNK - 1) / GP_BOP_ADD_CHUNK;
  if (n_chunks > 65535) return fail(GP_ERR_INVALID, "an object of %d vertices has more than 65535 chunks", max_v);
  if (!obj_idx || !vertices || !K || !frame_idx || !pose_est || !pose_gt || !workspace || !out)
    return fail(GP_ERR_INVALID, "null argument");
  if (reinterpret_cast<uintptr_t>(workspace) % 8) return fail(GP_ERR_INVALID, "workspace must be 8-byte aligned");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  double* partial = static_cast<double*>(workspace);
  GP_CUDA(gp::launch_ex(add_kernel<false>, dim3(n_pairs, n_chunks), kThreads, 0, st, 1, false, n_objects, obj_idx, tab,
                        vertices, n_frames, K, frame_idx, pose_est, pose_gt, partial, nullptr, nullptr, nullptr));
  GP_CUDA(gp::launch_ex(add_finish_kernel, (unsigned)((3ll * n_pairs + kThreads - 1) / kThreads), kThreads, 0, st, 1,
                        false, n_pairs, n_chunks, n_objects, obj_idx, tab, n_frames, frame_idx,
                        static_cast<const double*>(partial), out));
  return GP_OK;
}

// gp_vis_vertex_errors (csrc/vis.cu) validates its arguments and launches add_kernel<true> through here
cudaError_t gp::launch_add_vertex_errors(int n_pairs, int n_objects, const int32_t* obj_idx,
                                         const int32_t* vertex_offsets, const float* vertices, const float* pose_est,
                                         const float* pose_gt, const uint8_t* symmetric, const int64_t* out_offsets,
                                         float* values, cudaStream_t st) {
  VertexTable tab;
  int max_v = 0;
  for (int o = 0; o <= GP_BOP_MAX_OBJECTS; ++o) tab.off[o] = o <= n_objects ? vertex_offsets[o] : 0;
  for (int o = 1; o <= n_objects; ++o) max_v = max(max_v, vertex_offsets[o] - vertex_offsets[o - 1]);
  const int n_chunks = (max_v + GP_BOP_ADD_CHUNK - 1) / GP_BOP_ADD_CHUNK;
  return gp::launch_ex(add_kernel<true>, dim3(n_pairs, n_chunks), kThreads, 0, st, 1, false, n_objects, obj_idx, tab,
                       vertices, 1, nullptr, nullptr, pose_est, pose_gt, nullptr, symmetric,
                       reinterpret_cast<const long long*>(out_offsets), values);
}

static bool check_offsets(const int32_t* off, int n) {
  if (off[0] != 0) return false;
  for (int i = 1; i <= n; ++i)
    if (off[i] < off[i - 1]) return false;
  return true;
}

extern "C" int gp_bop_match(int n_groups, int n_objects, int n_theta, const int32_t* est_offsets,
                            const int32_t* gt_offsets, const int32_t* group_obj, const double* thresholds,
                            const float* mssd, const float* mspd, const uint8_t* gt_valid, void* workspace,
                            int8_t* labels, void* stream) {
  if (n_groups < 1) return fail(GP_ERR_INVALID, "n_groups %d must be >= 1", n_groups);
  if (n_objects < 1 || n_objects > GP_BOP_MAX_OBJECTS)
    return fail(GP_ERR_INVALID, "n_objects %d outside [1, %d]", n_objects, GP_BOP_MAX_OBJECTS);
  if (n_theta < 1 || n_theta > GP_BOP_MAX_TAU)
    return fail(GP_ERR_INVALID, "n_theta %d outside [1, %d]", n_theta, GP_BOP_MAX_TAU);
  if (!est_offsets || !gt_offsets || !group_obj || !thresholds) return fail(GP_ERR_INVALID, "null host table");
  if (!check_offsets(est_offsets, n_groups) || !check_offsets(gt_offsets, n_groups))
    return fail(GP_ERR_INVALID, "bad offsets: they must start at 0 and not decrease");
  const size_t n_thr = (size_t)n_objects * 2 * n_theta;
  for (size_t i = 0; i < n_thr; ++i)
    if (!isfinite(thresholds[i])) return fail(GP_ERR_INVALID, "thresholds[%zu] is not finite", i);
  if (!mssd || !mspd || !gt_valid || !workspace || !labels) return fail(GP_ERR_INVALID, "null argument");
  if (reinterpret_cast<uintptr_t>(workspace) % 8) return fail(GP_ERR_INVALID, "workspace must be 8-byte aligned");
  std::vector<unsigned char> host(n_thr * sizeof(double) + (size_t)n_groups * sizeof(MatchGroup));
  memcpy(host.data(), thresholds, n_thr * sizeof(double));
  MatchGroup* tab = reinterpret_cast<MatchGroup*>(host.data() + n_thr * sizeof(double));
  long long err0 = 0;
  for (int g = 0; g < n_groups; ++g) {
    const int n_gt = gt_offsets[g + 1] - gt_offsets[g];
    if (n_gt > GP_BOP_MAX_GT_PER_GROUP)
      return fail(GP_ERR_INVALID, "group %d has %d ground truths, more than %d", g, n_gt, GP_BOP_MAX_GT_PER_GROUP);
    if (group_obj[g] < 0 || group_obj[g] >= n_objects)
      return fail(GP_ERR_INVALID, "group_obj[%d] = %d outside [0, %d)", g, group_obj[g], n_objects);
    tab[g] = MatchGroup{err0, est_offsets[g], est_offsets[g + 1] - est_offsets[g], gt_offsets[g], n_gt, group_obj[g], 0};
    err0 += (long long)tab[g].n_est * n_gt;
  }
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GP_CUDA(cudaMemcpyAsync(workspace, host.data(), host.size(), cudaMemcpyHostToDevice, st));
  const double* thr_dev = static_cast<const double*>(workspace);
  const MatchGroup* tab_dev = reinterpret_cast<const MatchGroup*>(static_cast<const unsigned char*>(workspace) +
                                                                  n_thr * sizeof(double));
  const long long n_warps = (long long)n_groups * 2 * n_theta;
  GP_CUDA(gp::launch_ex(match_kernel, (unsigned)((n_warps + kWarps - 1) / kWarps), kThreads, 0, st, 1, false, n_warps,
                        n_theta, tab_dev, thr_dev, mssd, mspd, gt_valid, labels));
  return GP_OK;
}

extern "C" int gp_bop_average_precision(int n_objects, int n_theta, int n_est, const int8_t* labels,
                                        const int32_t* rank_offsets, const int32_t* rank, const int32_t* n_valid,
                                        int n_recall, const double* recall_thresholds, double* ap, void* stream) {
  if (n_objects < 1 || n_objects > GP_BOP_MAX_OBJECTS)
    return fail(GP_ERR_INVALID, "n_objects %d outside [1, %d]", n_objects, GP_BOP_MAX_OBJECTS);
  if (n_theta < 1 || n_theta > GP_BOP_MAX_TAU)
    return fail(GP_ERR_INVALID, "n_theta %d outside [1, %d]", n_theta, GP_BOP_MAX_TAU);
  if (n_est < 1) return fail(GP_ERR_INVALID, "n_est %d must be >= 1", n_est);
  if (n_recall < 1 || n_recall > GP_BOP_MAX_RECALL)
    return fail(GP_ERR_INVALID, "n_recall %d outside [1, %d]", n_recall, GP_BOP_MAX_RECALL);
  if (!rank_offsets || !n_valid || !recall_thresholds) return fail(GP_ERR_INVALID, "null host table");
  if (!check_offsets(rank_offsets, n_objects))
    return fail(GP_ERR_INVALID, "bad rank offsets: they must start at 0 and not decrease");
  ApTables tab;
  for (int o = 0; o <= GP_BOP_MAX_OBJECTS; ++o) tab.rank_off[o] = rank_offsets[min(o, n_objects)];
  for (int o = 0; o < GP_BOP_MAX_OBJECTS; ++o) {
    tab.n_valid[o] = o < n_objects ? n_valid[o] : 1;
    if (tab.n_valid[o] < 1) return fail(GP_ERR_INVALID, "n_valid[%d] = %d must be >= 1", o, tab.n_valid[o]);
  }
  for (int k = 0; k < GP_BOP_MAX_RECALL; ++k) {
    tab.recall[k] = k < n_recall ? recall_thresholds[k] : 0.0;
    if (k < n_recall && !isfinite(tab.recall[k]))
      return fail(GP_ERR_INVALID, "recall_thresholds[%d] is not finite", k);
    if (k > 0 && k < n_recall && tab.recall[k] < tab.recall[k - 1])
      return fail(GP_ERR_INVALID, "recall_thresholds must not decrease (at %d)", k);
  }
  if (!labels || !rank || !ap) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(ap_kernel, n_objects * 2 * n_theta, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false,
                        n_theta, n_est, labels, rank, n_recall, tab, ap));
  return GP_OK;
}
