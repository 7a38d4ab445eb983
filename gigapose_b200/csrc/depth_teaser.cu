// Row f13: depth refinement with MegaPose's TeaserppRefiner (src/megapose/inference/teaserpp_refiner.py:165-291, the
// sibling of the ICP of depth_icp.cu), on the GPU.  One hypothesis is a (detection, pose) pair with: the measured depth
// D [H,W] of its frame (the unit of the pose translations, mm for BOP; 0 = missing), the frame's full-image K, the
// coarse pose T0 and the depth R [H,W] of the object rendered at T0 with that K (gp_render_templates).  The reference's
// constants are in metres and scaled by `unit_per_m` (u): noise = noise_bound * u and eps2 = noise^2 in the pose unit.
// This file is compiled with -fmad=false (build.py), so every floating-point operation below rounds once, as written.
//
// Contract (what tests/test_gpu_teaser.py pins against oracle/teaser_port.py):
//  1. Points (teaser_points_kernel).  mask = (D > 0) & (R > 0) ("simple", refiner_utils.py:42-46).  The masked pixels
//     are compacted in row-major order within the render box (R is 0 outside it), so index 0 is the first masked pixel
//     in row-major order, as the reference's boolean indexing gives.  Back-projection (get_pointcloud): with the pixel
//     indices u, v and q = fp32(d / fx) (an fp32 division, as numpy divides an f32 image by an f32 scalar),
//     x = fp32(fp64(u - cx) * fp64(q)), y likewise with v, cy, fy, z = d.  Source points come from R, target points
//     from D.  N = the number of masked pixels; N < min_points (or N = 0): status TOO_FEW_POINTS.
//  2. Farthest-point sampling (teaser_fps_kernel) of M = min(n_points, N) source points: index 0 first, then for each
//     next sample the point with the largest min over the samples of the fp32 squared distance
//     ((dx dx + dy dy) + dz dz), d = p - sample; on a tie the lowest index.  The sampled indices apply to both clouds.
//     Deviation: the reference asks pytorch3d for K = n_points samples, padded with -1 (the last point) when N < K;
//     here M = N distinct samples are taken (INTEGRATION.md).  Whether pytorch3d breaks ties the same way is unverified.
//  3. Consistency graph, sampled points i < j: edge iff | ||t_j - t_i|| - ||s_j - s_i|| | <= 2 noise sqrt(cbar2), in
//     fp64: d = double(p_j) - double(p_i), l = sqrt((d0 d0 + d1 d1) + d2 d2), the bound 2 * noise * sqrt(cbar2).  The
//     bit-packed adjacency, 32 words of 32 bits per row, stays in shared memory (at most 1024 rows, 128 KiB).
//  4. Exact maximum clique.  Order: vertices by degree descending, the lower index first on a tie (positions 0 ..
//     M-1).  Lower bound: the greedy clique that adds the lowest-position candidate until none is left.  Search:
//     branch and bound over candidate sets P in position space; every visit of a node colours P greedily (classes
//     built in position order, each taking the lowest-position vertex not adjacent to the class); with k colours and
//     clique size d, d + k <= best prunes the node; otherwise the last vertex coloured, v, is branched on: the child is
//     P & N(v); a child that is empty is a maximal clique, kept when larger than the best; then v leaves P and P is
//     coloured again.  The best clique is the first one found of maximum size in this order.  Every node visit counts
//     against clique_budget; past it the status is CLIQUE_BUDGET.  A clique of fewer than 3: CLIQUE_TOO_SMALL.
//  5. Rotation: GNC-TLS over the chain TIMs of the clique's members c_0 < .. < c_{m-1} (sample indices):
//     s_k = double(s_{c_{k+1}}) - double(s_{c_k}) and t_k likewise, k + 1 taken mod m.  Weights w = 1; iteration i:
//     S_ab = sum_k (w_k s_ka) t_kb (the sums below), R = the rotation of Horn's quaternion (the eigenvector of the
//     largest eigenvalue, lowest index on a tie, of his 4 x 4 matrix of S; 8 cyclic Jacobi sweeps) -- a proper
//     rotation by construction; r_k = ||t_k - R s_k||^2 (rows ((R_a0 s0 + R_a1 s1) + R_a2 s2), then
//     (e0 e0 + e1 e1) + e2 e2).  At i = 0: mu = 1 / ((2 max r) / eps2 - 1), and the loop ends when mu is not > 0 or
//     not finite.  th1 = ((mu + 1) / mu) eps2, th2 = (mu / (mu + 1)) eps2; w_k = 0 if r_k >= th1, 1 if r_k <= th2,
//     else sqrt(((eps2 mu) (mu + 1)) / r_k) - mu; cost = sum_k w_k r_k with the new weights; mu *= gnc_factor; the
//     loop ends after gnc_max_iters iterations or when |cost - previous cost| < gnc_cost_threshold u^2.
//     Sums over k run per lane l over k = l, l + 32, .. in order, then across lanes by an xor butterfly (16, 8, 4, 2, 1).
//  6. Translation, per axis a: x_i = double(t_{c_i,a}) - (R s_{c_i})_a over the members, r = noise sqrt(cbar2).  The
//     2m endpoints (x_i - r, +(i+1)) and (x_i + r, -(i+1)) are sorted by value, then by the signed index; a sweep keeps
//     the consensus count n, sum x, sum x^2 and the outside range sum rs (starting at m r, summed in order), and for
//     n > 0 takes mean = sum x / n and cost = (((n mean) mean + sum x^2) - (2 sum x) mean) + u rs (u^2 times the
//     reference's cost in metres); t_a = the mean at the lowest cost, the first on a tie.
//  7. Inliers over the M samples: ||R s + t - t_i|| < noise (strict; ((R_a0 x + R_a1 y) + R_a2 z) + t_a, the norm as
//     in 5).  inliers >= min_inliers: out_pose = [R | t] T0 (fp64 rows ((T_a0 T0_0b + T_a1 T0_1b) + T_a2 T0_2b) +
//     T_a3 T0_3b, stored fp32), status OK.  Every other outcome returns T0 bit for bit with its status.
//
// Layout: three kernels, each one CTA per hypothesis: compaction and sampling (1024 threads), and the solve (512
// threads, ~193 KiB of shared memory: graph and order on the CTA, clique on warp 0 with one 32-bit word of each
// 1024-bit set per lane, GNC-TLS on warp 0, voting and inliers on the CTA).  A hypothesis' result depends on its own
// inputs only.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

#include <cmath>

using gp::fail;

namespace {

constexpr int kThreads = 1024;
constexpr int kWarps = kThreads / 32;
constexpr int kSolve = 512;                // the solve kernel: 128 registers per thread for the fp64 eigen solve
constexpr int kSolveWarps = kSolve / 32;
constexpr int kMaxPts = GP_TEASER_MAX_POINTS;      // 1024 = 32 words of 32 bits: one word per lane
constexpr int kWords = kMaxPts / 32;
constexpr int kMaxSide = 8192;
constexpr int kSweeps = 8;

struct Ws {               // per-call workspace, carved in this order
  float* pts;             // [n_hyp][6][H*W] compacted source x, y, z, target x, y, z
  float* mind;            // [n_hyp][H*W] FPS running minimum distances
  int* hdr;               // [n_hyp][4] N (-1: invalid frame)
  int* samples;           // [n_hyp][kMaxPts]
  uint32_t* stack;        // [n_hyp][kMaxPts + 1][kWords] the candidate set of each clique-search level
  uint32_t* perm;         // [n_hyp][kMaxPts][kWords] the adjacency in position space, before it goes to shared memory
};

Ws carve(void* base, int n_hyp, size_t plane) {
  gp::Carver c(base);
  Ws w;
  w.pts = c.take<float>((size_t)n_hyp * 6 * plane);
  w.mind = c.take<float>((size_t)n_hyp * plane);
  w.hdr = c.take<int>((size_t)n_hyp * 4);
  w.samples = c.take<int>((size_t)n_hyp * kMaxPts);
  w.stack = c.take<uint32_t>((size_t)n_hyp * (kMaxPts + 1) * kWords);
  w.perm = c.take<uint32_t>((size_t)n_hyp * kMaxPts * kWords);
  return w;
}

size_t carved_bytes(int n_hyp, size_t plane) {
  gp::Carver c(nullptr);
  c.take<float>((size_t)n_hyp * 6 * plane);
  c.take<float>((size_t)n_hyp * plane);
  c.take<int>((size_t)n_hyp * 4);
  c.take<int>((size_t)n_hyp * kMaxPts);
  c.take<uint32_t>((size_t)n_hyp * (kMaxPts + 1) * kWords);
  c.take<uint32_t>((size_t)n_hyp * kMaxPts * kWords);
  return c.off;
}

struct Box {
  int x0, y0, x1, y1;
};

__device__ __forceinline__ Box clip_box(const long long* b, int H, int W) {
  Box r;
  r.x0 = (int)max(0ll, min((long long)W, b[0]));
  r.y0 = (int)max(0ll, min((long long)H, b[1]));
  r.x1 = (int)max(0ll, min((long long)W, b[2]));
  r.y1 = (int)max(0ll, min((long long)H, b[3]));
  return r;
}

// --- 1. mask and compaction ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
teaser_points_kernel(int n_frames, int H, int W, const int32_t* __restrict__ frame_idx, const float* __restrict__ depth,
                     const float* __restrict__ rendered, const long long* __restrict__ boxes,
                     const float* __restrict__ K, Ws ws, float* __restrict__ dbg_points) {
  __shared__ int warp_tot[kWarps];
  __shared__ int warp_off[kWarps + 1];
  const int h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f = frame_idx[h];
  if (f < 0 || f >= n_frames) {
    if (tid == 0) ws.hdr[4 * h] = -1;
    return;
  }
  const size_t plane = (size_t)H * W;
  const float* dm = depth + f * plane;
  const float* dr = rendered + h * plane;
  const float fx = K[9 * f + 0], cx = K[9 * f + 2], fy = K[9 * f + 4], cy = K[9 * f + 5];
  const Box b = clip_box(boxes + 4 * h, H, W);
  const int bw = max(b.x1 - b.x0, 0), n = bw * max(b.y1 - b.y0, 0);
  float* pts = ws.pts + (size_t)h * 6 * plane;
  int base = 0;
  for (int p0 = 0; p0 < n; p0 += kThreads) {
    const int p = p0 + tid;
    bool keep = false;
    int u = 0, v = 0;
    float r = 0.f, m = 0.f;
    if (p < n) {
      v = b.y0 + p / bw;
      u = b.x0 + p % bw;
      r = dr[(size_t)v * W + u];
      m = dm[(size_t)v * W + u];
      keep = m > 0.f && r > 0.f;
    }
    const unsigned bal = __ballot_sync(0xffffffffu, keep);
    if (lane == 0) warp_tot[warp] = __popc(bal);
    __syncthreads();
    if (tid == 0) {
      int s = 0;
      for (int w = 0; w < kWarps; ++w) { warp_off[w] = s; s += warp_tot[w]; }
      warp_off[kWarps] = s;
    }
    __syncthreads();
    if (keep) {
      const size_t i = (size_t)base + warp_off[warp] + __popc(bal & ((1u << lane) - 1u));
      const double du = (double)u - (double)cx, dv = (double)v - (double)cy;
      const float xs = (float)(du * (double)(r / fx)), ys = (float)(dv * (double)(r / fy));
      const float xt = (float)(du * (double)(m / fx)), yt = (float)(dv * (double)(m / fy));
      pts[i] = xs; pts[plane + i] = ys; pts[2 * plane + i] = r;
      pts[3 * plane + i] = xt; pts[4 * plane + i] = yt; pts[5 * plane + i] = m;
      if (dbg_points) {
        float* o = dbg_points + ((size_t)h * plane + i) * 6;
        o[0] = xs; o[1] = ys; o[2] = r; o[3] = xt; o[4] = yt; o[5] = m;
      }
    }
    base += warp_off[kWarps];
    __syncthreads();                     // warp_off is rewritten by the next pass
  }
  if (tid == 0) ws.hdr[4 * h] = base;
}

// --- 2. farthest-point sampling ------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
teaser_fps_kernel(int H, int W, int min_points, int n_points, Ws ws) {
  __shared__ unsigned long long red[kWarps];
  __shared__ int sel_s;
  const int h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = ws.hdr[4 * h];
  if (N < min_points || N < 1) return;
  const size_t plane = (size_t)H * W;
  const float* px = ws.pts + (size_t)h * 6 * plane;
  const float *py = px + plane, *pz = px + 2 * plane;
  float* mind = ws.mind + (size_t)h * plane;
  int* samples = ws.samples + (size_t)h * kMaxPts;
  const int M = min(n_points, N);
  for (int i = tid; i < N; i += kThreads) mind[i] = __int_as_float(0x7f800000);
  if (tid == 0) samples[0] = 0;
  int sel = 0;
  for (int k = 1; k < M; ++k) {
    const float sx = px[sel], sy = py[sel], sz = pz[sel];
    unsigned long long best = 0;
    for (int i = tid; i < N; i += kThreads) {
      const float dx = px[i] - sx, dy = py[i] - sy, dz = pz[i] - sz;
      const float d = fminf(mind[i], (dx * dx + dy * dy) + dz * dz);
      mind[i] = d;
      const unsigned long long key = ((unsigned long long)__float_as_uint(d) << 32) | (0xffffffffu - (unsigned)i);
      best = key > best ? key : best;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
      best = x > best ? x : best;
    }
    if (lane == 0) red[warp] = best;
    __syncthreads();
    if (warp == 0) {
      best = red[lane];
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const unsigned long long x = __shfl_xor_sync(0xffffffffu, best, o);
        best = x > best ? x : best;
      }
      if (lane == 0) {
        sel_s = (int)(0xffffffffu - (unsigned)(best & 0xffffffffu));
        samples[k] = sel_s;
      }
    }
    __syncthreads();
    sel = sel_s;
  }
}

// --- 3-7. graph, clique, rotation, translation, inliers ------------------------------------------------------------
struct Smem {
  uint32_t adj[kMaxPts * kWords];   // vertex space, then position space
  float sp[3][kMaxPts], tp[3][kMaxPts];
  double w[kMaxPts];                // GNC weights
  double xv[kMaxPts];               // GNC residuals, then the translation votes of one axis
  int sorted[2 * kMaxPts];          // vote endpoints in sorted order
  int deg[kMaxPts];
  short vert[kMaxPts];              // position -> vertex
  short cur[kMaxPts], best[kMaxPts];
  short members[kMaxPts];           // clique members (vertices) ascending
  uint32_t cl[kWords];
  int red[kSolveWarps];
  double R[9], t[3];
  int m, status, best_size, iters;
  long long nodes;
};

__device__ __forceinline__ double butterfly(double v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v = v + __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ int first_bit(uint32_t word) {       // warp-wide: the lowest set bit of the lane words
  const unsigned b = __ballot_sync(0xffffffffu, word != 0u);
  if (!b) return -1;
  const int ln = __ffs(b) - 1;
  const uint32_t w = __shfl_sync(0xffffffffu, word, ln);
  return ln * 32 + __ffs(w) - 1;
}

// Horn's quaternion of S (S_ab = sum s_a t_b), the rotation taking s to t: the eigenvector of the largest eigenvalue of
// his 4 x 4 matrix, by kSweeps cyclic Jacobi sweeps (pairs in order (0,1) (0,2) (0,3) (1,2) (1,3) (2,3); a pair with an
// exact 0 off-diagonal entry is skipped).  oracle/teaser_port.py `horn` restates it operation for operation.
__device__ void horn(const double* S, double* R) {
  const double xx = S[0], xy = S[1], xz = S[2], yx = S[3], yy = S[4], yz = S[5], zx = S[6], zy = S[7], zz = S[8];
  double A[4][4] = {{(xx + yy) + zz, yz - zy, zx - xz, xy - yx},
                    {yz - zy, (xx - yy) - zz, xy + yx, zx + xz},
                    {zx - xz, xy + yx, (yy - xx) - zz, yz + zy},
                    {xy - yx, zx + xz, yz + zy, (zz - xx) - yy}};
  double V[4][4] = {{1, 0, 0, 0}, {0, 1, 0, 0}, {0, 0, 1, 0}, {0, 0, 0, 1}};
  for (int sw = 0; sw < kSweeps; ++sw)
    for (int p = 0; p < 3; ++p)
      for (int q = p + 1; q < 4; ++q) {
        const double apq = A[p][q];
        if (apq == 0.0) continue;
        const double th = (A[q][q] - A[p][p]) / (2.0 * apq);
        const double tt = (th >= 0.0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        const double c = 1.0 / sqrt(tt * tt + 1.0), s = tt * c;
        for (int k = 0; k < 4; ++k) {
          const double akp = A[k][p], akq = A[k][q];
          A[k][p] = c * akp - s * akq;
          A[k][q] = s * akp + c * akq;
        }
        for (int k = 0; k < 4; ++k) {
          const double apk = A[p][k], aqk = A[q][k];
          A[p][k] = c * apk - s * aqk;
          A[q][k] = s * apk + c * aqk;
        }
        for (int k = 0; k < 4; ++k) {
          const double vkp = V[k][p], vkq = V[k][q];
          V[k][p] = c * vkp - s * vkq;
          V[k][q] = s * vkp + c * vkq;
        }
      }
  int e = 0;
  for (int k = 1; k < 4; ++k)
    if (A[k][k] > A[e][e]) e = k;
  double qw = V[0][e], qx = V[1][e], qy = V[2][e], qz = V[3][e];
  const double nq = sqrt(((qw * qw + qx * qx) + qy * qy) + qz * qz);
  qw = qw / nq; qx = qx / nq; qy = qy / nq; qz = qz / nq;
  R[0] = ((qw * qw + qx * qx) - qy * qy) - qz * qz;
  R[1] = 2.0 * (qx * qy - qw * qz);
  R[2] = 2.0 * (qx * qz + qw * qy);
  R[3] = 2.0 * (qx * qy + qw * qz);
  R[4] = ((qw * qw - qx * qx) + qy * qy) - qz * qz;
  R[5] = 2.0 * (qy * qz - qw * qx);
  R[6] = 2.0 * (qx * qz - qw * qy);
  R[7] = 2.0 * (qy * qz + qw * qx);
  R[8] = ((qw * qw - qx * qx) - qy * qy) + qz * qz;
}

__device__ __forceinline__ double sqnorm_res(const double* R, const double* s, const double* t) {
  const double e0 = t[0] - ((R[0] * s[0] + R[1] * s[1]) + R[2] * s[2]);
  const double e1 = t[1] - ((R[3] * s[0] + R[4] * s[1]) + R[5] * s[2]);
  const double e2 = t[2] - ((R[6] * s[0] + R[7] * s[1]) + R[8] * s[2]);
  return (e0 * e0 + e1 * e1) + e2 * e2;
}

__global__ void __launch_bounds__(kSolve)
teaser_solve_kernel(int H, int W, gp_teaser_params_t p, const float* __restrict__ T0, float* __restrict__ out_poses,
                    int32_t* __restrict__ out_status, int32_t* __restrict__ out_inliers,
                    int32_t* __restrict__ out_clique, Ws ws) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  Smem& S = *reinterpret_cast<Smem*>(smem_raw);
  const int h = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const gp_teaser_debug_t& dbg = p.debug;
  const int N = ws.hdr[4 * h];
  const float* t0 = T0 + 16 * h;
  int status = GP_TEASER_OK, inliers = 0, clique = 0;
  const double noise = (double)p.noise_bound * (double)p.unit_per_m, eps2 = noise * noise;
  const int M = N > 0 ? min(p.n_points, N) : 0;
  if (dbg.counts && tid == 0) {
    int32_t* c = dbg.counts + 4 * h;
    c[0] = N; c[1] = N < p.min_points ? 0 : M; c[2] = 0; c[3] = 0;
  }
  if (N < 0) {
    status = GP_TEASER_INVALID;
  } else if (N < p.min_points || N < 1) {
    status = GP_TEASER_TOO_FEW_POINTS;
  } else if (p.debug.stop_after == 1 || p.debug.stop_after == 2) {
    status = -1;
  } else {
    const size_t plane = (size_t)H * W;
    const float* pts = ws.pts + (size_t)h * 6 * plane;
    const int* samples = ws.samples + (size_t)h * kMaxPts;
    for (int k = tid; k < M; k += kSolve) {
      const int i = samples[k];
#pragma unroll
      for (int a = 0; a < 3; ++a) {
        S.sp[a][k] = pts[a * plane + i];
        S.tp[a][k] = pts[(3 + a) * plane + i];
      }
      if (dbg.samples) dbg.samples[(size_t)h * p.n_points + k] = i;
    }
    __syncthreads();
    // 3. graph: thread task (row i, word w) tests the 32 columns of word w
    const double bound = (2.0 * noise) * sqrt((double)p.cbar2);
    for (int task = tid; task < M * kWords; task += kSolve) {
      const int i = task / kWords, w = task % kWords;
      const double si0 = S.sp[0][i], si1 = S.sp[1][i], si2 = S.sp[2][i];
      const double ti0 = S.tp[0][i], ti1 = S.tp[1][i], ti2 = S.tp[2][i];
      uint32_t bits = 0;
      for (int b = 0; b < 32; ++b) {
        const int j = w * 32 + b;
        if (j >= M || j == i) continue;
        const double a0 = (double)S.sp[0][j] - si0, a1 = (double)S.sp[1][j] - si1, a2 = (double)S.sp[2][j] - si2;
        const double b0 = (double)S.tp[0][j] - ti0, b1 = (double)S.tp[1][j] - ti1, b2 = (double)S.tp[2][j] - ti2;
        const double ls = sqrt((a0 * a0 + a1 * a1) + a2 * a2), lt = sqrt((b0 * b0 + b1 * b1) + b2 * b2);
        if (fabs(lt - ls) <= bound) bits |= 1u << b;
      }
      S.adj[i * kWords + w] = bits;
      if (dbg.adjacency) dbg.adjacency[((size_t)h * p.n_points + i) * kWords + w] = bits;
    }
    __syncthreads();
    // 4. order: degree descending, the lower index first
    for (int i = tid; i < M; i += kSolve) {
      int d = 0;
      for (int w = 0; w < kWords; ++w) d += __popc(S.adj[i * kWords + w]);
      S.deg[i] = d;
    }
    __syncthreads();
    for (int i = tid; i < M; i += kSolve) {
      const int di = S.deg[i];
      int r = 0;
      for (int j = 0; j < M; ++j) r += S.deg[j] > di || (S.deg[j] == di && j < i);
      S.vert[r] = (short)i;
    }
    __syncthreads();
    uint32_t* perm = ws.perm + (size_t)h * kMaxPts * kWords;
    for (int task = tid; task < M * kWords; task += kSolve) {
      const int pp = task / kWords, w = task % kWords;
      const int vi = S.vert[pp];
      uint32_t bits = 0;
      for (int b = 0; b < 32; ++b) {
        const int q = w * 32 + b;
        if (q >= M) break;
        const int vj = S.vert[q];
        bits |= ((S.adj[vi * kWords + (vj >> 5)] >> (vj & 31)) & 1u) << b;
      }
      perm[task] = bits;
    }
    __syncthreads();
    for (int task = tid; task < M * kWords; task += kSolve) S.adj[task] = perm[task];
    __syncthreads();
    if (p.debug.stop_after == 3) {
      status = -1;
    } else {
      if (warp == 0) {
        // 4. greedy lower bound, then branch and bound; lane l owns word l of every set
        const uint32_t full = lane * 32 >= M ? 0u : M - lane * 32 >= 32 ? 0xffffffffu : (1u << (M - lane * 32)) - 1u;
        uint32_t P = full;
        int bs = 0;
        for (int v = first_bit(P); v >= 0; v = first_bit(P)) {
          if (lane == 0) S.best[bs] = (short)v;
          ++bs;
          P &= S.adj[v * kWords + lane];
        }
        uint32_t* stk = ws.stack + (size_t)h * (kMaxPts + 1) * kWords;
        long long nodes = 0;
        bool over = false;
        int d = 0;
        P = full;
        stk[lane] = P;
        while (true) {
          if (++nodes > p.clique_budget) { over = true; break; }
          uint32_t Q = P;
          int k = 0, last = -1;
          while (__any_sync(0xffffffffu, Q != 0u)) {
            ++k;
            uint32_t Rr = Q;
            for (int v = first_bit(Rr); v >= 0; v = first_bit(Rr)) {
              Rr &= ~S.adj[v * kWords + lane];
              if ((v >> 5) == lane) { Rr &= ~(1u << (v & 31)); Q &= ~(1u << (v & 31)); }
              last = v;
            }
          }
          if (k == 0 || d + k <= bs) {
            if (d == 0) break;
            --d;
            P = stk[d * kWords + lane];
            const int v = S.cur[d];
            if ((v >> 5) == lane) P &= ~(1u << (v & 31));
            stk[d * kWords + lane] = P;
            continue;
          }
          const int v = last;
          if (lane == 0) S.cur[d] = (short)v;
          __syncwarp();
          const uint32_t NP = P & S.adj[v * kWords + lane];
          if (!__any_sync(0xffffffffu, NP != 0u)) {
            if (d + 1 > bs) {
              bs = d + 1;
              for (int k2 = lane; k2 < bs; k2 += 32) S.best[k2] = S.cur[k2];
            }
            if ((v >> 5) == lane) P &= ~(1u << (v & 31));
            stk[d * kWords + lane] = P;
            __syncwarp();
            continue;
          }
          ++d;
          P = NP;
          stk[d * kWords + lane] = P;
        }
        __syncwarp();
        if (lane == 0) {
          S.best_size = bs;
          S.nodes = nodes;
          S.status = over ? GP_TEASER_CLIQUE_BUDGET : bs < 3 ? GP_TEASER_CLIQUE_TOO_SMALL : GP_TEASER_OK;
        }
        // members ascending: bitset of their vertices, then a prefix count over the lanes
        S.cl[lane] = 0u;
        __syncwarp();
        for (int k2 = lane; k2 < bs; k2 += 32) {
          const int vv = S.vert[S.best[k2]];
          atomicOr(&S.cl[vv >> 5], 1u << (vv & 31));
        }
        __syncwarp();
        const uint32_t word = S.cl[lane];
        int off = __popc(word);
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int x = __shfl_up_sync(0xffffffffu, off, o);
          if (lane >= o) off += x;
        }
        off -= __popc(word);
        for (uint32_t wb = word; wb; wb &= wb - 1u) S.members[off++] = (short)(lane * 32 + __ffs(wb) - 1);
        if (lane == 0) S.m = bs;
      }
      __syncthreads();
      status = S.status;
      clique = S.best_size;
      const int m = S.m;
      if (dbg.counts && tid == 0) dbg.counts[4 * h + 2] = (int)min(S.nodes, 0x7fffffffll);
      if (dbg.clique)
        for (int k = tid; k < p.n_points; k += kSolve)
          dbg.clique[(size_t)h * p.n_points + k] = status == GP_TEASER_OK && k < m ? S.members[k] : -1;
      if (status == GP_TEASER_OK && p.debug.stop_after == 4) status = -1;
      if (status == GP_TEASER_OK) {
        // 5. GNC-TLS rotation over the chain TIMs, on warp 0
        if (warp == 0) {
          for (int k = lane; k < m; k += 32) S.w[k] = 1.0;
          __syncwarp();
          double prev = __longlong_as_double(0x7ff0000000000000ll), mu = 0.0, R[9];
          const double thr = (double)p.gnc_cost_threshold * ((double)p.unit_per_m * (double)p.unit_per_m);
          int it = 0;
          for (; it < p.gnc_max_iters;) {
            double Sm[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
            for (int k = lane; k < m; k += 32) {
              const int a = S.members[k], b = S.members[k + 1 == m ? 0 : k + 1];
              const double wk = S.w[k];
              double s[3], t[3];
#pragma unroll
              for (int c = 0; c < 3; ++c) {
                s[c] = (double)S.sp[c][b] - (double)S.sp[c][a];
                t[c] = (double)S.tp[c][b] - (double)S.tp[c][a];
              }
#pragma unroll
              for (int c = 0; c < 3; ++c) {
                const double ws_ = wk * s[c];
#pragma unroll
                for (int e = 0; e < 3; ++e) Sm[3 * c + e] = Sm[3 * c + e] + ws_ * t[e];
              }
            }
#pragma unroll
            for (int c = 0; c < 9; ++c) Sm[c] = butterfly(Sm[c]);
            horn(Sm, R);
            const bool trace = dbg.gnc && it < dbg.gnc_capacity;
            if (trace && dbg.gnc_weights)
              for (int k = lane; k < m; k += 32)
                dbg.gnc_weights[((size_t)h * dbg.gnc_capacity + it) * p.n_points + k] = S.w[k];
            double maxr = 0.0;
            for (int k = lane; k < m; k += 32) {
              const int a = S.members[k], b = S.members[k + 1 == m ? 0 : k + 1];
              double s[3], t[3];
#pragma unroll
              for (int c = 0; c < 3; ++c) {
                s[c] = (double)S.sp[c][b] - (double)S.sp[c][a];
                t[c] = (double)S.tp[c][b] - (double)S.tp[c][a];
              }
              const double r = sqnorm_res(R, s, t);
              S.xv[k] = r;
              maxr = fmax(maxr, r);
            }
#pragma unroll
            for (int o = 16; o; o >>= 1) maxr = fmax(maxr, __shfl_xor_sync(0xffffffffu, maxr, o));
            __syncwarp();
            bool stop = false;
            if (it == 0) {
              mu = 1.0 / ((2.0 * maxr) / eps2 - 1.0);
              stop = !(mu > 0.0) || isinf(mu);
            }
            double cost = 0.0;
            if (!stop) {
              const double th1 = ((mu + 1.0) / mu) * eps2, th2 = (mu / (mu + 1.0)) * eps2;
              for (int k = lane; k < m; k += 32) {
                const double r = S.xv[k];
                const double wk = r >= th1 ? 0.0 : r <= th2 ? 1.0 : sqrt(((eps2 * mu) * (mu + 1.0)) / r) - mu;
                S.w[k] = wk;
                cost = cost + wk * r;
              }
              cost = butterfly(cost);
            }
            if (trace && lane == 0) {
              gp_teaser_gnc_t& g = dbg.gnc[(size_t)h * dbg.gnc_capacity + it];
              g.iteration = it;
              g.members = m;
              g.stopped = stop ? 1 : 0;
              g.reserved = 0;
              g.mu = mu;
              g.cost = cost;
              g.max_residual = maxr;
              for (int c = 0; c < 9; ++c) g.R[c] = R[c];
            }
            ++it;
            if (stop) break;
            const double diff = fabs(cost - prev);
            mu = mu * (double)p.gnc_factor;
            prev = cost;
            __syncwarp();
            if (diff < thr) break;
          }
          if (lane == 0) {
            for (int c = 0; c < 9; ++c) S.R[c] = R[c];
            S.iters = it;
          }
        }
        __syncthreads();
        if (dbg.counts && tid == 0) dbg.counts[4 * h + 3] = S.iters;
        double R[9];
        for (int c = 0; c < 9; ++c) R[c] = S.R[c];
        // 6. adaptive voting per axis
        const double r = noise * sqrt((double)p.cbar2);
        const int n2 = 2 * m;
        for (int a = 0; a < 3; ++a) {
          for (int k = tid; k < m; k += kSolve) {
            const int i = S.members[k];
            const double s0 = S.sp[0][i], s1 = S.sp[1][i], s2 = S.sp[2][i];
            S.xv[k] = (double)S.tp[a][i] - ((R[3 * a] * s0 + R[3 * a + 1] * s1) + R[3 * a + 2] * s2);
          }
          __syncthreads();
          for (int e = tid; e < n2; e += kSolve) {
            const double ve = (e & 1) ? S.xv[e >> 1] + r : S.xv[e >> 1] - r;
            const int se = (e & 1) ? -((e >> 1) + 1) : (e >> 1) + 1;
            int rank = 0;
            for (int g = 0; g < n2; ++g) {
              const double vg = (g & 1) ? S.xv[g >> 1] + r : S.xv[g >> 1] - r;
              const int sg = (g & 1) ? -((g >> 1) + 1) : (g >> 1) + 1;
              rank += vg < ve || (vg == ve && sg < se);
            }
            S.sorted[rank] = e;
          }
          __syncthreads();
          if (tid == 0) {
            int cnt = 0;
            double sx = 0.0, sxx = 0.0, rs = 0.0, best = __longlong_as_double(0x7ff0000000000000ll), est = 0.0;
            for (int k = 0; k < m; ++k) rs = rs + r;
            for (int q = 0; q < n2; ++q) {
              const int e = S.sorted[q];
              const double x = S.xv[e >> 1];
              if (e & 1) { --cnt; sx = sx - x; sxx = sxx - x * x; rs = rs + r; }
              else { ++cnt; sx = sx + x; sxx = sxx + x * x; rs = rs - r; }
              if (cnt > 0) {
                const double mean = sx / (double)cnt;
                const double cost = ((((double)cnt * mean) * mean + sxx) - (2.0 * sx) * mean) + (double)p.unit_per_m * rs;
                if (cost < best) { best = cost; est = mean; }
              }
            }
            S.t[a] = est;
          }
          __syncthreads();
        }
        const double t[3] = {S.t[0], S.t[1], S.t[2]};
        if (dbg.transform && tid == 0) {
          double* o = dbg.transform + 12 * (size_t)h;
          for (int c = 0; c < 9; ++c) o[c] = R[c];
          for (int c = 0; c < 3; ++c) o[9 + c] = t[c];
        }
        // 7. inliers over the M samples
        int cnt = 0;
        for (int k = tid; k < M; k += kSolve) {
          const double s0 = S.sp[0][k], s1 = S.sp[1][k], s2 = S.sp[2][k];
          const double e0 = ((R[0] * s0 + R[1] * s1) + R[2] * s2) + t[0] - (double)S.tp[0][k];
          const double e1 = ((R[3] * s0 + R[4] * s1) + R[5] * s2) + t[1] - (double)S.tp[1][k];
          const double e2 = ((R[6] * s0 + R[7] * s1) + R[8] * s2) + t[2] - (double)S.tp[2][k];
          cnt += sqrt((e0 * e0 + e1 * e1) + e2 * e2) < noise;
        }
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        if (lane == 0) S.red[warp] = cnt;
        __syncthreads();
        inliers = 0;
        for (int w = 0; w < kSolveWarps; ++w) inliers += S.red[w];
        if (inliers < p.min_inliers) status = GP_TEASER_TOO_FEW_INLIERS;
        if (status == GP_TEASER_OK && tid == 0) {
          const double T[12] = {R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]};
          for (int a = 0; a < 3; ++a)
            for (int b = 0; b < 4; ++b)
              out_poses[16 * h + 4 * a + b] =
                  (float)((((T[4 * a] * (double)t0[b] + T[4 * a + 1] * (double)t0[4 + b]) + T[4 * a + 2] * (double)t0[8 + b]) +
                           T[4 * a + 3] * (double)t0[12 + b]));
          for (int b = 0; b < 4; ++b) out_poses[16 * h + 12 + b] = t0[12 + b];
        }
      }
    }
  }
  if (tid == 0) {
    if (status != GP_TEASER_OK)
      for (int c = 0; c < 16; ++c) out_poses[16 * h + c] = t0[c];
    out_status[h] = status;
    out_inliers[h] = inliers;
    out_clique[h] = clique;
  }
}

int check_params(const gp_teaser_params_t* p) {
  if (!p) return fail(GP_ERR_INVALID, "null params");
  if (!(p->unit_per_m > 0.f) || !std::isfinite(p->unit_per_m)) return fail(GP_ERR_INVALID, "unit_per_m must be > 0");
  if (p->n_points < 3 || p->n_points > kMaxPts)
    return fail(GP_ERR_INVALID, "n_points %d outside [3, %d]", p->n_points, kMaxPts);
  if (p->min_points < 1) return fail(GP_ERR_INVALID, "min_points %d must be >= 1", p->min_points);
  if (!(p->noise_bound > 0.f) || !std::isfinite(p->noise_bound))
    return fail(GP_ERR_INVALID, "noise_bound must be finite and > 0");
  if (!(p->cbar2 > 0.f) || !std::isfinite(p->cbar2)) return fail(GP_ERR_INVALID, "cbar2 must be finite and > 0");
  if (p->min_inliers < 0) return fail(GP_ERR_INVALID, "min_inliers %d must be >= 0", p->min_inliers);
  if (!(p->gnc_factor > 1.f) || !std::isfinite(p->gnc_factor)) return fail(GP_ERR_INVALID, "gnc_factor must be > 1");
  if (p->gnc_max_iters < 1) return fail(GP_ERR_INVALID, "gnc_max_iters %d must be >= 1", p->gnc_max_iters);
  if (!(p->gnc_cost_threshold >= 0.0)) return fail(GP_ERR_INVALID, "gnc_cost_threshold must be >= 0");
  if (p->clique_budget < 1) return fail(GP_ERR_INVALID, "clique_budget must be >= 1");
  if (p->debug.gnc && p->debug.gnc_capacity < 1) return fail(GP_ERR_INVALID, "debug.gnc needs gnc_capacity >= 1");
  if (p->debug.gnc_weights && !p->debug.gnc) return fail(GP_ERR_INVALID, "debug.gnc_weights needs debug.gnc");
  if (p->debug.stop_after < 0 || p->debug.stop_after > 4)
    return fail(GP_ERR_INVALID, "debug.stop_after %d outside [0, 4]", p->debug.stop_after);
  return GP_OK;
}

int check_size(int n_hyp, int height, int width) {
  if (n_hyp < 1) return fail(GP_ERR_INVALID, "n_hyp %d must be >= 1", n_hyp);
  if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [1, %d]", height, width, kMaxSide);
  return GP_OK;
}

}  // namespace

extern "C" int gp_teaser_query_sizes(int n_hyp, int height, int width, size_t* workspace_bytes) {
  if (int e = check_size(n_hyp, height, width)) return e;
  if (!workspace_bytes) return fail(GP_ERR_INVALID, "null workspace_bytes");
  *workspace_bytes = carved_bytes(n_hyp, (size_t)height * width);
  return GP_OK;
}

extern "C" int gp_teaser_refine(int n_frames, int n_hyp, int height, int width, const int32_t* frame_idx,
                                const float* depth, const float* rendered_depth, const int64_t* boxes, const float* T0,
                                const float* K, const gp_teaser_params_t* params, float* out_poses,
                                int32_t* out_status, int32_t* out_inliers, int32_t* out_clique, void* workspace,
                                void* stream) {
  if (int e = check_size(n_hyp, height, width)) return e;
  if (n_frames < 1) return fail(GP_ERR_INVALID, "n_frames %d must be >= 1", n_frames);
  if (int e = check_params(params)) return e;
  if (!frame_idx || !depth || !rendered_depth || !boxes || !T0 || !K || !out_poses || !out_status || !out_inliers ||
      !out_clique || !workspace)
    return fail(GP_ERR_INVALID, "null argument");
  if (reinterpret_cast<uintptr_t>(workspace) % gp::kAlign)
    return fail(GP_ERR_INVALID, "workspace must be %zu-byte aligned", gp::kAlign);
  const gp_teaser_params_t p = *params;
  const Ws ws = carve(workspace, n_hyp, (size_t)height * width);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const long long* bx = reinterpret_cast<const long long*>(boxes);
  GP_CUDA(gp::launch_ex(teaser_points_kernel, n_hyp, kThreads, 0, st, 1, false, n_frames, height, width, frame_idx,
                        depth, rendered_depth, bx, K, ws, p.debug.points));
  if (p.debug.stop_after != 1)
    GP_CUDA(gp::launch_ex(teaser_fps_kernel, n_hyp, kThreads, 0, st, 1, false, height, width, p.min_points,
                          p.n_points, ws));
  GP_CUDA(gp::launch_ex(teaser_solve_kernel, n_hyp, kSolve, sizeof(Smem), st, 1, false, height, width, p, T0,
                        out_poses, out_status, out_inliers, out_clique, ws));
  return GP_OK;
}
