// Exhaustive one-point RANSAC, hypothesis scoring/sorting and 6-D pose lifting for sm_90a
// (rows a7-a9 of SURVEY.md §8; replaces RANSAC.forward/forward_ ransac.py:37-172, ObjectPoseRecovery.forward_ransac /
// forward_recovery poses.py:26-163, the affine helpers lib3d/torch.py:7-89,150-162 and gigaPose.py:588-604).
//
// The reference runs B*k python iterations, builds an [n, n-1] index on the CPU per iteration and syncs on every
// boolean mask.  Here one CTA handles one (detection, hypothesis): the valid correspondences are compacted in
// ascending patch order (that order is what torch.max's first-maximum tie-break sees), every candidate similarity
// transform is scored against all other correspondences from shared memory, and the inliers of the winner are
// compacted again.  fp32 arithmetic follows the reference's operation order (separate multiply/add, no FMA
// contraction) because the 14-pixel inlier test is a knife edge.
#include "gigapose_kernels.h"

namespace gp {

namespace {

constexpr int kP = 256;

// exclusive prefix count of `flag` over the 256 threads of the CTA (ascending thread order), plus total
__device__ __forceinline__ int block_scan_256(bool flag, int* s_warp, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned bal = __ballot_sync(0xffffffffu, flag);
  const int within = __popc(bal & ((1u << lane) - 1));
  __syncthreads();
  if (lane == 0) s_warp[warp] = __popc(bal);
  __syncthreads();
  int base = 0, tot = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) {
    const int c = s_warp[w];
    if (w < warp) base += c;
    tot += c;
  }
  total = tot;
  return base + within;
}

__global__ void __launch_bounds__(256)
ransac_kernel(RansacParams p) {
  __shared__ float s_sx[kP], s_sy[kP], s_tx[kP], s_ty[kP];     // pixel coordinates of the valid correspondences
  __shared__ int s_src[kP], s_tar[kP];                         // packed raw patch coordinates (x | y << 8)
  __shared__ float s_m00[kP], s_m01[kP], s_m10[kP], s_m11[kP], s_m02[kP], s_m12[kP];
  __shared__ int s_warp[8];
  __shared__ int s_bw_score[8], s_bw_idx[8];
  __shared__ int s_best;
  const int bk = blockIdx.x;
  const int t = threadIdx.x;
  const size_t base = (size_t)bk * kP;
  const long long sxi = p.src_pts[2 * (base + t)], syi = p.src_pts[2 * (base + t) + 1];
  const long long txi = p.tar_pts[2 * (base + t)], tyi = p.tar_pts[2 * (base + t) + 1];
  const bool valid = sxi != -1;                                 // ransac.py:141
  int n;
  const int pos = block_scan_256(valid, s_warp, n);
  const float ps = (float)p.patch_size;
  if (valid) {
    const float sx = (float)sxi * ps, sy = (float)syi * ps;     // ransac.py:57-58: pixel units, no half-patch offset
    const float tx = (float)txi * ps, ty = (float)tyi * ps;
    s_sx[pos] = sx; s_sy[pos] = sy; s_tx[pos] = tx; s_ty[pos] = ty;
    s_src[pos] = (int)sxi | ((int)syi << 8);
    s_tar[pos] = (int)txi | ((int)tyi << 8);
    const float sc = p.rel_scale[base + t];
    const float c = p.rel_inplane[2 * (base + t)], s = p.rel_inplane[2 * (base + t) + 1];
    // affine_torch (lib3d/torch.py:21-29): rotation [[c,-s],[s,c]] scaled element-wise
    const float m00 = __fmul_rn(c, sc), m01 = __fmul_rn(-s, sc), m10 = __fmul_rn(s, sc), m11 = __fmul_rn(c, sc);
    // apply_affine on the proposing point with zero translation (ransac.py:91-93)
    const float ax = __fadd_rn(__fadd_rn(__fmul_rn(m00, sx), __fmul_rn(m01, sy)), 0.0f);
    const float ay = __fadd_rn(__fadd_rn(__fmul_rn(m10, sx), __fmul_rn(m11, sy)), 0.0f);
    s_m00[pos] = m00; s_m01[pos] = m01; s_m10[pos] = m10; s_m11[pos] = m11;
    s_m02[pos] = __fsub_rn(tx, ax);
    s_m12[pos] = __fsub_rn(ty, ay);
  }
  // default outputs (ransac.py:129-135)
  p.in_score[base + t] = 0;
  p.in_src[2 * (base + t)] = -1; p.in_src[2 * (base + t) + 1] = -1;
  p.in_tar[2 * (base + t)] = -1; p.in_tar[2 * (base + t) + 1] = -1;
  __syncthreads();

  if (n == 0) {                                                 // ransac.py:142: nothing to fit, identity / not failed
    if (t < 9) p.M[(size_t)bk * 9 + t] = (t % 4 == 0) ? 1.f : 0.f;
    if (t == 0) { p.failed[bk] = 0; p.in_count[bk] = 0; }
    return;
  }

  // score candidate i = t against every other correspondence (ransac.py:96-99)
  const float thr = p.pixel_threshold;
  int score = -1;
  if (t < n) {
    const float m00 = s_m00[t], m01 = s_m01[t], m10 = s_m10[t], m11 = s_m11[t], m02 = s_m02[t], m12 = s_m12[t];
    score = 0;
    for (int j = 0; j < n; ++j) {
      if (j == t) continue;                                     // validation set excludes the proposer (ransac.py:29-33)
      const float px = __fadd_rn(__fadd_rn(__fmul_rn(m00, s_sx[j]), __fmul_rn(m01, s_sy[j])), m02);
      const float py = __fadd_rn(__fadd_rn(__fmul_rn(m10, s_sx[j]), __fmul_rn(m11, s_sy[j])), m12);
      const float dx = __fsub_rn(s_tx[j], px), dy = __fsub_rn(s_ty[j], py);
      const float err = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
      score += (err <= thr) ? 1 : 0;
    }
  }
  // first maximum over candidates in ascending order (torch.max, ransac.py:100)
  int bs = score, bi = t;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const int os = __shfl_xor_sync(0xffffffffu, bs, off);
    const int oi = __shfl_xor_sync(0xffffffffu, bi, off);
    if (os > bs || (os == bs && oi < bi)) { bs = os; bi = oi; }
  }
  if ((t & 31) == 0) { s_bw_score[t >> 5] = bs; s_bw_idx[t >> 5] = bi; }
  __syncthreads();
  if (t == 0) {
    for (int w = 1; w < 8; ++w)
      if (s_bw_score[w] > bs || (s_bw_score[w] == bs && s_bw_idx[w] < bi)) { bs = s_bw_score[w]; bi = s_bw_idx[w]; }
    s_best = bi;
    p.failed[bk] = (bs == 0) ? 1 : 0;                           // ransac.py:101
    p.in_count[bk] = bs;
    float* M = p.M + (size_t)bk * 9;
    M[0] = s_m00[bi]; M[1] = s_m01[bi]; M[2] = s_m02[bi];
    M[3] = s_m10[bi]; M[4] = s_m11[bi]; M[5] = s_m12[bi];
    M[6] = 0.f; M[7] = 0.f; M[8] = 1.f;
  }
  __syncthreads();
  // inliers of the winner, compacted in ascending order (ransac.py:104-105,159-162)
  const int best = s_best;
  bool inl = false;
  if (t < n && t != best) {
    const float px = __fadd_rn(__fadd_rn(__fmul_rn(s_m00[best], s_sx[t]), __fmul_rn(s_m01[best], s_sy[t])), s_m02[best]);
    const float py = __fadd_rn(__fadd_rn(__fmul_rn(s_m10[best], s_sx[t]), __fmul_rn(s_m11[best], s_sy[t])), s_m12[best]);
    const float dx = __fsub_rn(s_tx[t], px), dy = __fsub_rn(s_ty[t], py);
    inl = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) <= thr;
  }
  int cnt;
  const int ipos = block_scan_256(inl, s_warp, cnt);
  if (inl) {
    p.in_src[2 * (base + ipos)] = s_src[t] & 255;
    p.in_src[2 * (base + ipos) + 1] = s_src[t] >> 8;
    p.in_tar[2 * (base + ipos)] = s_tar[t] & 255;
    p.in_tar[2 * (base + ipos) + 1] = s_tar[t] >> 8;
    p.in_score[base + ipos] = 1;
  }
}

// ------------------------------------------------------------------------------------------------------------
// scores = inliers / 256, stable descending sort of the k hypotheses, permutation of every [B,k,...] tensor
// (gigaPose.py:588-595) and pose lifting of the sorted hypotheses (poses.py:26-122).  One CTA per detection.
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mat3_mul(const float* A, const float* B, float* C) {
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) C[i * 3 + j] = A[i * 3] * B[j] + A[i * 3 + 1] * B[3 + j] + A[i * 3 + 2] * B[6 + j];
}

// (template id, 2-D similarity M, crop matrices, intrinsics) -> 4x4 pose (poses.py:26-101)
__device__ __forceinline__ void lift_pose(const float* Kt, const float* Mt, const float* Pt, const float* M,
                                          const float* Kq, const float* Mq, float* out) {
  // in-plane rotation = first 2x2 block of M divided by the norm of its first column (lib3d/torch.py:150-162)
  const float sc = sqrtf(M[0] * M[0] + M[3] * M[3]);
  const float Rin[9] = {M[0] / sc, M[1] / sc, 0.f, M[3] / sc, M[4] / sc, 0.f, 0.f, 0.f, 1.f};
  float Rt[9], R[9];
#pragma unroll
  for (int i = 0; i < 3; ++i)
#pragma unroll
    for (int j = 0; j < 3; ++j) Rt[i * 3 + j] = Pt[i * 4 + j];
  mat3_mul(Rin, Rt, R);                                       // poses.py:69-71
  const float tz = Pt[11];
  // template centre projected with the template intrinsics (poses.py:74-77)
  float c[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) c[i] = Kt[i * 3] * Pt[3] + Kt[i * 3 + 1] * Pt[7] + Kt[i * 3 + 2] * Pt[11];
  const float cz = c[2];
  c[0] /= cz; c[1] /= cz; c[2] /= cz;
  // inverse of the scale+translation query crop matrix (lib3d/torch.py:47-65), then affine2d = Mq^-1 . M . Mt
  const float qs = Mq[0];
  const float Minv[9] = {1.f / qs, 0.f, -Mq[2] / qs, 0.f, 1.f / qs, -Mq[5] / qs, 0.f, 0.f, 1.f};
  float T1[9], A[9];
  mat3_mul(Minv, M, T1);
  mat3_mul(T1, Mt, A);
  float qc[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) qc[i] = A[i * 3] * c[0] + A[i * 3 + 1] * c[1] + A[i * 3 + 2] * c[2];
  // general 3x3 inverse of the query intrinsics (torch.inverse, poses.py:89)
  const float a = Kq[0], bb = Kq[1], cc = Kq[2], d = Kq[3], e = Kq[4], f = Kq[5], g = Kq[6], h = Kq[7], i9 = Kq[8];
  const float det = a * (e * i9 - f * h) - bb * (d * i9 - f * g) + cc * (d * h - e * g);
  const float id = 1.f / det;
  const float Ki[9] = {(e * i9 - f * h) * id, (cc * h - bb * i9) * id, (bb * f - cc * e) * id,
                       (f * g - d * i9) * id, (a * i9 - cc * g) * id, (cc * d - a * f) * id,
                       (d * h - e * g) * id, (bb * g - a * h) * id, (a * e - bb * d) * id};
  const float s2d = sqrtf(A[0] * A[0] + A[3] * A[3]);        // poses.py:92
  const float qz = (tz / s2d) * (Kq[0] / Kt[0]);              // poses.py:93-94
  float tr[3];
#pragma unroll
  for (int i = 0; i < 3; ++i) tr[i] = Ki[i * 3] * qc[0] + Ki[i * 3 + 1] * qc[1] + Ki[i * 3 + 2] * qc[2];
  const float trz = tr[2];
#pragma unroll
  for (int i = 0; i < 3; ++i) tr[i] = (tr[i] / trz) * qz;     // poses.py:97-99
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    out[i * 4 + 0] = R[i * 3 + 0]; out[i * 4 + 1] = R[i * 3 + 1]; out[i * 4 + 2] = R[i * 3 + 2]; out[i * 4 + 3] = tr[i];
  }
  out[12] = Pt[12]; out[13] = Pt[13]; out[14] = Pt[14]; out[15] = Pt[15];
}

__global__ void __launch_bounds__(256)
sort_and_pose_kernel(PoseParams p) {
  __shared__ int s_order[32];
  const int b = blockIdx.x, t = threadIdx.x, k = p.k;
  if (t == 0) {
    // stable insertion sort, descending by inlier count (== descending score)
    int cnt[32];
    for (int i = 0; i < k; ++i) { cnt[i] = p.in_count[(size_t)b * k + i]; s_order[i] = i; }
    for (int i = 1; i < k && p.sort; ++i) {
      const int oi = s_order[i], ci = cnt[oi];
      int j = i - 1;
      while (j >= 0 && cnt[s_order[j]] < ci) { s_order[j + 1] = s_order[j]; --j; }
      s_order[j + 1] = oi;
    }
  }
  __syncthreads();
  for (int kk = 0; kk < k; ++kk) {
    const size_t src = (size_t)b * k + s_order[kk], dst = (size_t)b * k + kk;
    // per-patch tensors
    p.o_score_pts[dst * kP + t] = p.score_pts[src * kP + t];
    p.o_rel_scale[dst * kP + t] = p.rel_scale[src * kP + t];
    reinterpret_cast<float2*>(p.o_rel_inplane)[dst * kP + t] = reinterpret_cast<const float2*>(p.rel_inplane)[src * kP + t];
    reinterpret_cast<longlong2*>(p.o_tar_pts)[dst * kP + t] = reinterpret_cast<const longlong2*>(p.tar_pts)[src * kP + t];
    reinterpret_cast<longlong2*>(p.o_src_pts)[dst * kP + t] = reinterpret_cast<const longlong2*>(p.src_pts)[src * kP + t];
    reinterpret_cast<longlong2*>(p.o_in_src)[dst * kP + t] = reinterpret_cast<const longlong2*>(p.in_src)[src * kP + t];
    reinterpret_cast<longlong2*>(p.o_in_tar)[dst * kP + t] = reinterpret_cast<const longlong2*>(p.in_tar)[src * kP + t];
    p.o_in_score[dst * kP + t] = p.in_score[src * kP + t];
    if (t < 9) p.o_M[dst * 9 + t] = p.M[src * 9 + t];
    if (t == 0) {
      p.o_id_src[dst] = p.id_src[src];
      p.o_score_src[dst] = p.score_src[src];
      p.o_failed[dst] = p.failed[src];
      p.o_scores[dst] = (float)p.in_count[src] / (float)kP;     // gigaPose.py:588
    }
  }
  // pose lifting of hypothesis kk = t (poses.py:26-101)
  if (t < k) {
    const size_t src = (size_t)b * k + s_order[t], dst = (size_t)b * k + t;
    const int o = p.q_obj[b];
    const long long view = p.id_src[src];
    lift_pose(p.tmpl_K + (size_t)o * 9, p.tmpl_M + ((size_t)o * p.T + view) * 9,
              p.tmpl_pose + ((size_t)o * p.T + view) * 16, p.M + src * 9, p.q_K + (size_t)b * 9, p.q_M + (size_t)b * 9,
              p.o_poses + dst * 16);
  }
}

// ObjectPoseRecovery.forward_recovery alone (poses.py:103-122): one thread per (detection, hypothesis)
__global__ void pose_only_kernel(int n, int k, int T, const int* __restrict__ q_obj, const float* __restrict__ q_K,
                                 const float* __restrict__ q_M, const long long* __restrict__ id_src,
                                 const float* __restrict__ M, const float* __restrict__ tmpl_K,
                                 const float* __restrict__ tmpl_M, const float* __restrict__ tmpl_pose,
                                 float* __restrict__ poses) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = i / k;
  const int o = q_obj[b];
  const long long view = id_src[i];
  lift_pose(tmpl_K + (size_t)o * 9, tmpl_M + ((size_t)o * T + view) * 9, tmpl_pose + ((size_t)o * T + view) * 16,
            M + (size_t)i * 9, q_K + (size_t)b * 9, q_M + (size_t)b * 9, poses + (size_t)i * 16);
}

}  // namespace

cudaError_t launch_ransac(const RansacParams& p, cudaStream_t stream) {
  if (p.n <= 0) return cudaSuccess;
  return launch_ex(ransac_kernel, p.n, 256, 0, stream, 1, false, p);
}

cudaError_t launch_pose_only(int n, int k, int T, const int* q_obj, const float* q_K, const float* q_M,
                             const long long* id_src, const float* M, const float* tmpl_K, const float* tmpl_M,
                             const float* tmpl_pose, float* poses, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  return launch_ex(pose_only_kernel, (n + 127) / 128, 128, 0, stream, 1, false, n, k, T, q_obj, q_K, q_M, id_src, M, tmpl_K,
                   tmpl_M, tmpl_pose, poses);
}

cudaError_t launch_sort_and_pose(const PoseParams& p, cudaStream_t stream) {
  if (p.B <= 0) return cudaSuccess;
  if (p.k > 32) return cudaErrorInvalidValue;
  return launch_ex(sort_and_pose_kernel, p.B, 256, 0, stream, 1, false, p);
}

}  // namespace gp
