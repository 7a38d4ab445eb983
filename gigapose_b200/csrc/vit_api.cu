// C-ABI of the native DINOv2 ViT-L/14 forward (include/gigapose_b200.h, gp_vit_*): weight packing into bf16 hi/lo
// planes, TMA descriptors, and the per-layer launch sequence.  Geometry is fixed to what the reference uses
// (configs/model/ae_net/dinov2_l.yaml): 224x224 crops, patch 14, dim 1024, 16 heads, MLP 4096; depth is a parameter
// (24 for ViT-L) so that small stacks can be parity-tested quickly.
#include "../../include/gigapose_b200.h"
#include "gigapose_kernels.h"

#include <memory>
#include <new>
#include <vector>

using gp::Carver;
using gp::fail;

namespace {

constexpr int kDim = 1024, kQkv = 3072, kMlp = 4096, kTok = 257, kPatchK = 588, kPatchKPad = 608;
constexpr float kLayerNormEps = 1e-6f;          // DINOv2's norm layers (nn.LayerNorm(eps=1e-6)); gp_debug_layernorm uses it too

struct Planes { uint16_t *hi, *lo; CUtensorMap m_hi, m_lo; };

struct BlockW {
  Planes qkv, proj, fc1, fc2;
  const float *n1w, *n1b, *qkv_b, *proj_b, *ls1, *n2w, *n2b, *fc1_b, *fc2_b, *ls2;
};

struct AttnMaps { CUtensorMap hi128, lo128, hi16, lo16; };   // attention operand tiles: 64 columns x {128,16} token rows

}  // namespace

struct gp_vit_context {
  int depth, max_crops, passes, num_sms;
  Planes patch_w;
  const float *patch_b, *cls, *pos;
  std::vector<BlockW> blocks;
  // workspace
  float* x;                    // [max_crops*257, 1024] residual stream
  Planes ln, qkv, attn, hid, patches;   // activation planes (+ TMA maps for those that feed a GEMM)
  AttnMaps qkv_maps;           // over the head-major QKV planes
  size_t workspace_bytes;
};

namespace {

void carve_weights(Carver& c, int depth, gp_vit_context* h) {
  auto planes = [&](Planes* p, size_t n) { uint16_t* a = c.take<uint16_t>(n); uint16_t* b = c.take<uint16_t>(n); if (p) { p->hi = a; p->lo = b; } };
  planes(h ? &h->patch_w : nullptr, (size_t)kDim * kPatchKPad);
  for (int i = 0; i < depth; ++i) {
    BlockW* b = h ? &h->blocks[i] : nullptr;
    planes(b ? &b->qkv : nullptr, (size_t)kQkv * kDim);
    planes(b ? &b->proj : nullptr, (size_t)kDim * kDim);
    planes(b ? &b->fc1 : nullptr, (size_t)kMlp * kDim);
    planes(b ? &b->fc2 : nullptr, (size_t)kDim * kMlp);
  }
}

void carve_workspace(Carver& c, int max_crops, gp_vit_context* h) {
  const size_t M = (size_t)max_crops * kTok;
  auto planes = [&](Planes* p, size_t n) { uint16_t* a = c.take<uint16_t>(n); uint16_t* b = c.take<uint16_t>(n); if (p) { p->hi = a; p->lo = b; } };
  float* x = c.take<float>(M * kDim);
  if (h) h->x = x;
  planes(h ? &h->ln : nullptr, M * kDim);
  planes(h ? &h->qkv : nullptr, M * kQkv);
  planes(h ? &h->attn : nullptr, M * kDim);
  planes(h ? &h->hid : nullptr, M * kMlp);
  planes(h ? &h->patches : nullptr, (size_t)max_crops * 256 * kPatchKPad);
}

int make_maps(Planes* p, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  if (int e = gp::make_map(&p->m_hi, p->hi, rows, cols, box_rows)) return e;
  return gp::make_map(&p->m_lo, p->lo, rows, cols, box_rows);
}

// attention operand maps over head-major QKV planes holding crop_stride crops: rows = 3 * crop_stride * 16 heads * 257
int make_attention_maps(AttnMaps* m, const uint16_t* qkv_hi, const uint16_t* qkv_lo, int crop_stride) {
  const uint64_t rows = 48ull * crop_stride * kTok;
  auto* hi = const_cast<uint16_t*>(qkv_hi);
  auto* lo = const_cast<uint16_t*>(qkv_lo);
  int e;
  (e = gp::make_map_ex(&m->hi128, hi, rows, 64, 64, 128, 128)) || (e = gp::make_map_ex(&m->lo128, lo, rows, 64, 64, 128, 128)) ||
      (e = gp::make_map_ex(&m->hi16, hi, rows, 64, 64, 16, 128)) || (e = gp::make_map_ex(&m->lo16, lo, rows, 64, 64, 16, 128));
  return e;
}

// One transformer block over b crops: LayerNorm, QKV, attention, proj (+LayerScale +residual), LayerNorm, FC1 (+GELU),
// FC2 (+LayerScale +residual).  linears_only issues just the four GEMMs, on whatever the planes hold.
int run_block(const gp_vit_context* h, const BlockW& B, int b, bool linears_only, cudaStream_t s) {
  const int M = b * kTok;
  auto params = [&](int N, int K, int mode, const float* bias) {
    gp::GemmParams g{};
    g.passes = h->passes; g.M = M; g.N = N; g.K = K; g.mode = mode; g.bias = bias;
    return g;
  };
  auto linear = [&](const Planes& a, const Planes& w, const gp::GemmParams& g) {
    return gp::launch_vit_gemm(a.m_hi, a.m_lo, w.m_hi, w.m_lo, g, h->num_sms, s);
  };
  gp::GemmParams qkv = params(kQkv, kDim, gp::GEMM_QKV_HEADS, B.qkv_b);
  qkv.out_hi = h->qkv.hi; qkv.out_lo = h->qkv.lo; qkv.tokens_per_img = kTok; qkv.qkv_crop_stride = h->max_crops;
  gp::GemmParams proj = params(kDim, kDim, gp::GEMM_SCALE_RESIDUAL, B.proj_b);
  proj.gamma = B.ls1; proj.x = h->x;
  gp::GemmParams fc1 = params(kMlp, kDim, gp::GEMM_PLANES_GELU, B.fc1_b);
  fc1.out_hi = h->hid.hi; fc1.out_lo = h->hid.lo;
  gp::GemmParams fc2 = params(kDim, kMlp, gp::GEMM_SCALE_RESIDUAL, B.fc2_b);
  fc2.gamma = B.ls2; fc2.x = h->x;
  const AttnMaps& am = h->qkv_maps;
  if (!linears_only) GP_CUDA(gp::launch_layernorm_planes(h->x, M, B.n1w, B.n1b, kLayerNormEps, h->ln.hi, h->ln.lo, s));
  GP_CUDA(linear(h->ln, B.qkv, qkv));
  if (!linears_only)
    GP_CUDA(gp::launch_attention_tc(am.hi128, am.lo128, am.hi16, am.lo16, h->qkv.hi, h->qkv.lo, h->attn.hi, h->attn.lo, b,
                                    h->max_crops, h->passes, s));
  GP_CUDA(linear(h->attn, B.proj, proj));
  if (!linears_only) GP_CUDA(gp::launch_layernorm_planes(h->x, M, B.n2w, B.n2b, kLayerNormEps, h->ln.hi, h->ln.lo, s));
  GP_CUDA(linear(h->ln, B.fc1, fc1));
  GP_CUDA(linear(h->hid, B.fc2, fc2));
  return GP_OK;
}

}  // namespace

extern "C" {

int gp_vit_query_sizes(int depth, int max_crops, size_t* weight_bytes, size_t* workspace_bytes) {
  if (depth < 1 || depth > 64 || max_crops < 1) return fail(GP_ERR_INVALID, "bad depth / max_crops");
  Carver cw(nullptr), cs(nullptr);
  carve_weights(cw, depth, nullptr);
  carve_workspace(cs, max_crops, nullptr);
  if (weight_bytes) *weight_bytes = cw.off;
  if (workspace_bytes) *workspace_bytes = cs.off;
  return GP_OK;
}

int gp_vit_create(int device, int depth, int max_crops, int precision, const float* const* w, void* weight_mem,
                  void* workspace_mem, void* stream, gp_vit_handle_t* out) {
  if (depth < 1 || depth > 64 || max_crops < 1 || !w || !weight_mem || !workspace_mem || !out)
    return fail(GP_ERR_INVALID, "bad argument");
  if (precision != GP_PRECISION_FP32_SPLIT && precision != GP_PRECISION_BF16)
    return fail(GP_ERR_INVALID, "unknown precision %d", precision);
  if (((uintptr_t)weight_mem | (uintptr_t)workspace_mem) & (gp::kAlign - 1))
    return fail(GP_ERR_INVALID, "weight and workspace memory must be 1024-byte aligned");
  for (int i = 0; i < 4 + 14 * depth; ++i)
    if (!w[i]) return fail(GP_ERR_INVALID, "weight pointer %d is null", i);
  int num_sms = 0;
  if (int e = gp::open_device(device, &num_sms)) return e;
  std::unique_ptr<gp_vit_context> h(new (std::nothrow) gp_vit_context());
  if (!h) return fail(GP_ERR_INVALID, "out of host memory");
  h->depth = depth; h->max_crops = max_crops; h->num_sms = num_sms;
  h->passes = precision == GP_PRECISION_FP32_SPLIT ? 3 : 1;
  h->blocks.resize(depth);
  Carver cw(weight_mem), cs(workspace_mem);
  carve_weights(cw, depth, h.get());
  carve_workspace(cs, max_crops, h.get());
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // activation planes start finite: the attention tiles read up to 15 token rows past a crop (masked keys, P = 0),
  // and 0 * NaN from never-written memory would poison the P.V accumulation
  GP_CUDA(cudaMemsetAsync(workspace_mem, 0, cs.off, s));

  // pack weights: fp32 [N,K] -> bf16 hi/lo planes (patch embedding padded 588 -> 608 columns)
  h->patch_b = w[1]; h->cls = w[2]; h->pos = w[3];
  GP_CUDA(gp::launch_split_planes(w[0], kDim, kPatchK, kPatchKPad, h->patch_w.hi, h->patch_w.lo, s));
  if (int e = make_maps(&h->patch_w, kDim, kPatchKPad, 256)) return e;
  for (int i = 0; i < depth; ++i) {
    const float* const* b = w + 4 + 14 * i;
    BlockW& B = h->blocks[i];
    B.n1w = b[0]; B.n1b = b[1]; B.qkv_b = b[3]; B.proj_b = b[5]; B.ls1 = b[6];
    B.n2w = b[7]; B.n2b = b[8]; B.fc1_b = b[10]; B.fc2_b = b[12]; B.ls2 = b[13];
    GP_CUDA(gp::launch_split_planes(b[2], kQkv, kDim, kDim, B.qkv.hi, B.qkv.lo, s));
    GP_CUDA(gp::launch_split_planes(b[4], kDim, kDim, kDim, B.proj.hi, B.proj.lo, s));
    GP_CUDA(gp::launch_split_planes(b[9], kMlp, kDim, kDim, B.fc1.hi, B.fc1.lo, s));
    GP_CUDA(gp::launch_split_planes(b[11], kDim, kMlp, kMlp, B.fc2.hi, B.fc2.lo, s));
    int e;
    if ((e = make_maps(&B.qkv, kQkv, kDim, 256)) || (e = make_maps(&B.proj, kDim, kDim, 256)) ||
        (e = make_maps(&B.fc1, kMlp, kDim, 256)) || (e = make_maps(&B.fc2, kDim, kMlp, 256)))
      return e;
  }
  const uint64_t M = (uint64_t)max_crops * kTok;
  int e;
  if ((e = make_maps(&h->ln, M, kDim, 128)) || (e = make_maps(&h->attn, M, kDim, 128)) || (e = make_maps(&h->hid, M, kMlp, 128)) ||
      (e = make_maps(&h->patches, (uint64_t)max_crops * 256, kPatchKPad, 128)) ||
      (e = make_attention_maps(&h->qkv_maps, h->qkv.hi, h->qkv.lo, max_crops)))
    return e;
  *out = h.release();
  return GP_OK;
}

int gp_debug_attention_timeline(long long* stamps32) {
  if (!stamps32) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(cudaDeviceSynchronize());
  GP_CUDA(gp::read_attention_stamps(stamps32));
  return GP_OK;
}

int gp_debug_gemm_timeline(long long* stamps128) {
  if (!stamps128) return fail(GP_ERR_INVALID, "null argument");
  GP_CUDA(cudaDeviceSynchronize());
  GP_CUDA(gp::read_gemm_stamps(stamps128));
  return GP_OK;
}

int gp_debug_gemm(const gp_debug_gemm_t* d, void* stream) {
  if (!d) return fail(GP_ERR_INVALID, "null argument");
  gp::GemmParams g{};
  g.M = d->M; g.N = d->N; g.K = d->K; g.bn = d->bn; g.passes = d->passes; g.mode = d->mode; g.swap = d->swap; g.f16 = d->f16;
  g.acc_scale = d->acc_scale; g.bias = d->bias; g.gamma = d->gamma; g.x = d->x; g.out_hi = d->out_hi; g.out_lo = d->out_lo;
  g.pos = d->pos; g.res_hi = d->res_hi; g.res_lo = d->res_lo; g.m_dev = d->m_dev;
  g.tokens_per_img = d->tokens_per_img; g.patches_per_img = d->patches_per_img; g.qkv_crop_stride = d->qkv_crop_stride;
  g.stamp = d->stamp;
  if (g.M < 1) return fail(GP_ERR_INVALID, "M must be >= 1");
  const char* why = nullptr;
  if (!gp::gemm_config_supported(g, &why)) return fail(GP_ERR_INVALID, "unsupported GEMM: %s", why);
  if (!d->a_hi || !d->a_lo || !d->w_hi || !d->w_lo || !d->bias) return fail(GP_ERR_INVALID, "null operand or bias");
  const bool planes_out = g.mode == gp::GEMM_PLANES || g.mode == gp::GEMM_PLANES_GELU || g.mode == gp::GEMM_QKV_HEADS ||
                          g.mode == gp::GEMM_PLANES_RELU || g.mode == gp::GEMM_PLANES_ADD_RELU;
  if (planes_out ? (!g.out_hi || !g.out_lo) : !g.x) return fail(GP_ERR_INVALID, "null output");
  if (g.mode == gp::GEMM_SCALE_RESIDUAL && !g.gamma) return fail(GP_ERR_INVALID, "null gamma");
  if (g.mode == gp::GEMM_PLANES_ADD_RELU && (!g.res_hi || !g.res_lo)) return fail(GP_ERR_INVALID, "null residual planes");
  if (g.mode == gp::GEMM_PATCH_EMBED && (!g.pos || g.patches_per_img < 1 || g.tokens_per_img <= g.patches_per_img))
    return fail(GP_ERR_INVALID, "patch embedding needs pos and tokens_per_img > patches_per_img >= 1");
  if (g.mode == gp::GEMM_QKV_HEADS && (g.N != kQkv || g.tokens_per_img < 1 || g.qkv_crop_stride * g.tokens_per_img < g.M))
    return fail(GP_ERR_INVALID, "QKV scatter needs N = 3072 and qkv_crop_stride * tokens_per_img >= M");
  if (g.swap && g.m_dev) return fail(GP_ERR_INVALID, "m_dev is not supported with swap");
  int dev = 0, sms = 0;
  GP_CUDA(cudaGetDevice(&dev));
  GP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const int bn = g.bn > 0 ? g.bn : 256;
  // A: 128-row boxes; W: bn-row boxes (the swapped form streams 256 output pixels as its W operand)
  CUtensorMap a_hi, a_lo, w_hi, w_lo;
  auto* a_h = const_cast<uint16_t*>(d->a_hi); auto* a_l = const_cast<uint16_t*>(d->a_lo);
  auto* w_h = const_cast<uint16_t*>(d->w_hi); auto* w_l = const_cast<uint16_t*>(d->w_lo);
  if (int e = gp::make_map(&a_hi, a_h, g.M, g.K, 128)) return e;
  if (int e = gp::make_map(&a_lo, a_l, g.M, g.K, 128)) return e;
  if (int e = gp::make_map(&w_hi, w_h, g.N, g.K, bn)) return e;
  if (int e = gp::make_map(&w_lo, w_l, g.N, g.K, bn)) return e;
  GP_CUDA(gp::launch_vit_gemm(a_hi, a_lo, w_hi, w_lo, g, sms, static_cast<cudaStream_t>(stream)));
  return GP_OK;
}

int gp_debug_attention(int b, int crop_stride, int passes, const uint16_t* qkv_hi, const uint16_t* qkv_lo, uint16_t* out_hi,
                       uint16_t* out_lo, void* stream) {
  if (!qkv_hi || !qkv_lo || !out_hi || !out_lo) return fail(GP_ERR_INVALID, "null argument");
  if (b < 1 || crop_stride < b) return fail(GP_ERR_INVALID, "need 1 <= b (%d) <= crop_stride (%d)", b, crop_stride);
  if (passes != 1 && passes != 3) return fail(GP_ERR_INVALID, "passes must be 1 or 3");
  AttnMaps m;
  if (int e = make_attention_maps(&m, qkv_hi, qkv_lo, crop_stride)) return e;
  GP_CUDA(gp::launch_attention_tc(m.hi128, m.lo128, m.hi16, m.lo16, qkv_hi, qkv_lo, out_hi, out_lo, b, crop_stride, passes,
                                  static_cast<cudaStream_t>(stream)));
  return GP_OK;
}

int gp_debug_layernorm(int M, const float* x, const float* w, const float* b, uint16_t* out_hi, uint16_t* out_lo,
                       void* stream) {
  if (!x || !w || !b || !out_hi || !out_lo) return fail(GP_ERR_INVALID, "null argument");
  if (M < 1) return fail(GP_ERR_INVALID, "M must be >= 1");
  GP_CUDA(gp::launch_layernorm_planes(x, M, w, b, kLayerNormEps, out_hi, out_lo, static_cast<cudaStream_t>(stream)));
  return GP_OK;
}

int gp_vit_destroy(gp_vit_handle_t h) {
  delete h;
  return GP_OK;
}

// diagnostics: the 4 * depth linear layers of one forward over `b` crops, back to back on `stream`, `iters` times,
// between two CUDA events (synchronises the stream).  Operands are whatever the workspace holds (the GEMM does not
// care); the residual stream is clobbered and rebuilt by the next gp_vit_forward.
int gp_vit_time_linears(gp_vit_handle_t h, int b, int iters, float* avg_ms, void* stream) {
  if (!h || !avg_ms || iters < 1) return fail(GP_ERR_INVALID, "bad argument");
  if (b < 1 || b > h->max_crops) return fail(GP_ERR_INVALID, "batch %d outside [1, %d]", b, h->max_crops);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return gp::time_runs(s, iters, avg_ms, [&]() -> int {
    for (const BlockW& B : h->blocks)
      if (int e = run_block(h, B, b, true, s)) return e;
    return GP_OK;
  });
}

int gp_vit_forward(gp_vit_handle_t h, int b, const float* img, float* x_prenorm, void* stream) {
  if (!h || !img || !x_prenorm) return fail(GP_ERR_INVALID, "null argument");
  if (b < 1 || b > h->max_crops) return fail(GP_ERR_INVALID, "batch %d outside [1, %d]", b, h->max_crops);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int M = b * kTok;
  // patch embedding: im2col -> GEMM (+bias +pos) into token rows 1..256 of every crop; CLS rows separately
  GP_CUDA(gp::launch_im2col(img, b, kPatchKPad, h->patches.hi, h->patches.lo, s));
  gp::GemmParams g{};
  g.passes = h->passes; g.tokens_per_img = kTok; g.patches_per_img = 256;
  g.M = b * 256; g.N = kDim; g.K = kPatchKPad; g.mode = gp::GEMM_PATCH_EMBED; g.bias = h->patch_b; g.pos = h->pos; g.x = h->x;
  GP_CUDA(gp::launch_vit_gemm(h->patches.m_hi, h->patches.m_lo, h->patch_w.m_hi, h->patch_w.m_lo, g, h->num_sms, s));
  GP_CUDA(gp::launch_cls_rows(h->cls, h->pos, b, h->x, s));
  for (const BlockW& B : h->blocks)
    if (int e = run_block(h, B, b, false, s)) return e;
  GP_CUDA(cudaMemcpyAsync(x_prenorm, h->x, (size_t)M * kDim * sizeof(float), cudaMemcpyDeviceToDevice, s));
  return GP_OK;
}

}  // extern "C"
