// Row f10: the depth-consistency score that ranks the refined hypotheses of a detection.  The reference keeps the best
// of its refined hypotheses with MegaPose's learned coarse model (src/megapose/inference/pose_estimator.py:580-623);
// with a measured depth image the render of each final pose can be compared with it pixel by pixel instead, in the
// spirit of VSD's visibility test (Hodan et al., "BOP: Benchmark for 6D Object Pose Estimation", ECCV 2018), with no
// weights.  The host side (gigapose_b200/icp.py, score_hypotheses) renders the poses with the renderer call the ICP's
// sources come from and calls gp_depth_score.
//
// Contract (what tests/test_gpu_depth_score.py pins against oracle/depth_score_port.py, bit for bit):
//  gp_depth_score, one 256-thread CTA per detection d, walking the render boxes of its hypotheses i = d * n_hyp + j,
//  j = 0 .. n_hyp - 1, in order.  A box is [x0, y0, x1, y1) as gp_render_templates writes it, clipped to the image; a
//  box that is empty after clipping (x1 <= x0 or y1 <= y0) contributes nothing and no pixel of it is read.  For every
//  pixel of the box with r = rendered[i] > 0 there, and m the measured depth of frame frame_idx[d] there:
//    !(m > 0)                       -> missing   (0, negative and NaN are all "no measurement")
//    __fsub_rn(m, r) > tolerance    -> behind    (the camera sees through the model: the claimed surface is not there)
//    __fsub_rn(r, m) > tolerance    -> front     (something is in front of the model: occluded)
//    otherwise                      -> consistent
//  counts i32 [n_det * n_hyp, 4] = (consistent, behind, front, missing);
//  score = __fdiv_rn(float(consistent), float(consistent + behind + front)), 0 when the denominator is 0 (an empty
//  render, or no measured pixel under it); each integer is converted to fp32 with one rounding (exact below 2^24).
//  best[d] = the j with the largest score, the lowest j on a tie, so the coarse order decides when depth cannot.
//  A detection whose frame index is outside [0, n_frames) gets counts -1, scores NaN (bits 0x7fffffff) and best -1.
//  Per-thread integer counts, __reduce_add_sync per warp, the warps summed in a fixed order by thread 0, which also
//  keeps the running best: every output is an integer or one rounded division, independent of the schedule.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

#include <cmath>

using gp::fail;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxSide = 8192;

__global__ void __launch_bounds__(kThreads)
depth_score_kernel(int n_frames, int n_hyp, int H, int W, const int32_t* __restrict__ frame_idx,
                   const float* __restrict__ depth, const float* __restrict__ rendered,
                   const long long* __restrict__ boxes, float tolerance, int32_t* __restrict__ counts,
                   float* __restrict__ score, int32_t* __restrict__ best) {
  __shared__ int red[kWarps][4];
  const int d = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int f = frame_idx[d];
  if (f < 0 || f >= n_frames) {
    for (int c = tid; c < 4 * n_hyp; c += kThreads) counts[(size_t)d * n_hyp * 4 + c] = -1;
    for (int c = tid; c < n_hyp; c += kThreads) score[(size_t)d * n_hyp + c] = __int_as_float(0x7fffffff);
    if (tid == 0) best[d] = -1;
    return;
  }
  const size_t plane = (size_t)H * W;
  const float* dm = depth + f * plane;
  int best_j = 0;
  float best_score = -1.f;                // thread 0 only; every score is >= 0, so hypothesis 0 always replaces it
  for (int j = 0; j < n_hyp; ++j) {
    const size_t i = (size_t)d * n_hyp + j;
    const long long* b = boxes + 4 * i;
    const int x0 = (int)max(0ll, min((long long)W, b[0])), y0 = (int)max(0ll, min((long long)H, b[1]));
    const int x1 = (int)max(0ll, min((long long)W, b[2])), y1 = (int)max(0ll, min((long long)H, b[3]));
    const float* dr = rendered + i * plane;
    int cnt[4] = {0, 0, 0, 0};
    const int bw = max(x1 - x0, 0), n = bw * max(y1 - y0, 0);
    for (int p = tid; p < n; p += kThreads) {
      const size_t q = (size_t)(y0 + p / bw) * W + (x0 + p % bw);
      const float r = dr[q];
      if (r > 0.f) {
        const float m = dm[q];
        const int c = !(m > 0.f) ? 3 : __fsub_rn(m, r) > tolerance ? 1 : __fsub_rn(r, m) > tolerance ? 2 : 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) cnt[k] += c == k;
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int s = __reduce_add_sync(0xffffffffu, cnt[k]);
      if (lane == 0) red[warp][k] = s;
    }
    __syncthreads();
    if (tid == 0) {
      int tot[4] = {0, 0, 0, 0};
      for (int w = 0; w < kWarps; ++w)
#pragma unroll
        for (int k = 0; k < 4; ++k) tot[k] += red[w][k];
#pragma unroll
      for (int k = 0; k < 4; ++k) counts[4 * i + k] = tot[k];
      const int den = tot[0] + tot[1] + tot[2];
      const float s = den == 0 ? 0.f : __fdiv_rn((float)tot[0], (float)den);
      score[i] = s;
      if (s > best_score) {
        best_score = s;
        best_j = j;
      }
    }
    __syncthreads();                      // red is rewritten by the next hypothesis
  }
  if (tid == 0) best[d] = best_j;
}

}  // namespace

extern "C" int gp_depth_score(int n_frames, int n_det, int n_hyp, int height, int width, const int32_t* frame_idx,
                              const float* depth, const float* rendered, const int64_t* boxes, float tolerance,
                              int32_t* counts, float* score, int32_t* best, void* stream) {
  if (n_frames < 1 || n_det < 1 || n_hyp < 1)
    return fail(GP_ERR_INVALID, "n_frames %d, n_det %d, n_hyp %d must be >= 1", n_frames, n_det, n_hyp);
  if (height < 1 || width < 1 || height > kMaxSide || width > kMaxSide)
    return fail(GP_ERR_INVALID, "image size %d x %d outside [1, %d]", height, width, kMaxSide);
  if (!(tolerance >= 0.f) || !std::isfinite(tolerance))
    return fail(GP_ERR_INVALID, "tolerance must be finite and not negative");
  if (!frame_idx || !depth || !rendered || !boxes || !counts || !score || !best)
    return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(gp::launch_ex(depth_score_kernel, n_det, kThreads, 0, static_cast<cudaStream_t>(stream), 1, false, n_frames,
                        n_hyp, height, width, frame_idx, depth, rendered, reinterpret_cast<const long long*>(boxes),
                        tolerance, counts, score, best));
  return GP_OK;
}
