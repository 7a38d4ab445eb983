/*
 * gigapose_b200 -- C ABI of the H100-native GigaPose inference hot path (libgigapose_b200.so).
 *
 * The reference (nv-nguyen/gigapose) is pure Python: it has no FFI.  Its boundary for this path is a set of
 * Python classes resolved by Hydra `_target_` strings (configs/model/large.yaml:1,36;
 * configs/model/ae_net/dinov2_l.yaml:1; configs/model/ist_net/resnet.yaml:1,6,16).  The Python mirror of those
 * classes lives in this repository under `src/` and calls the entry points below through ctypes
 * (gigapose_b200/_lib.py); each entry point cites the reference code it replaces.
 *
 * Conventions
 *  - every function returns 0 on success or a negative gp_status; gp_last_error() gives the message
 *    (thread local);  no C++ exceptions cross the boundary;
 *  - all tensor pointers are DEVICE pointers owned by the caller; dense, row-major, the dtypes stated below;
 *  - all work is enqueued on the caller's `stream` (a cudaStream_t passed as void*); no call synchronises the
 *    host and no call allocates device memory: the bank and the workspace are caller-provided at gp_create and
 *    sized by gp_query_sizes;
 *  - one handle per (thread, GPU); a handle is not thread safe.
 */
#ifndef GIGAPOSE_B200_H_
#define GIGAPOSE_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GP_ABI_VERSION 2
#define GP_NUM_PATCHES 256   /* 16 x 16 patches of a 224 x 224 crop, patch size 14 */
#define GP_AE_DIM 1024       /* DINOv2 ViT-L/14 descriptor size (configs/model/ae_net/dinov2_l.yaml:10) */
#define GP_IST_DIM 256       /* IST descriptor size (configs/model/ist_net/resnet.yaml:3) */
/* largest num_templates per handle: the top-k selection keeps one float per template in the 48 KiB of shared memory a
 * kernel gets without opting in, minus 1 KiB left for its static shared memory: (48 - 1) KiB / 4 B */
#define GP_MAX_NUM_TEMPLATES 12032

typedef enum gp_status {
  GP_OK = 0,
  GP_ERR_INVALID = -1,       /* bad argument / configuration */
  GP_ERR_CUDA = -2,          /* a CUDA runtime / driver call failed */
  GP_ERR_UNSUPPORTED = -3,   /* not an sm_90 device, or driver without TMA descriptor support */
  GP_ERR_STATE = -4          /* call order violated (e.g. search before queries were set) */
} gp_status;

typedef struct gp_context* gp_handle_t;

/* feature layouts accepted by gp_bank_write / gp_set_queries */
#define GP_LAYOUT_CHANNEL_MAJOR 0   /* [n, C, 16, 16]  -- what the reference modules exchange (ae_net.py:49-53) */
#define GP_LAYOUT_PATCH_MAJOR 1     /* [n, 256, C]     -- ViT token order, kernel-native                       */
#define GP_LAYOUT_VIT_TOKENS 2      /* [n, 257, C]     -- raw `x_prenorm` of gp_vit_forward: the CLS row of every crop is
                                       skipped (ae_net.py:65); use norm_passes = 2 (ae_net.py:69 + matching.py:229)   */

/* precision of the similarity contraction */
#define GP_PRECISION_FP32_SPLIT 0   /* bf16 hi/lo planes, hi*hi + hi*lo + lo*hi on tensor cores: fp32-faithful indices */
#define GP_PRECISION_BF16 1         /* hi*hi only: plain bf16 tensor-core similarity (3x less tensor work)       */

typedef struct gp_config {
  int32_t abi_version;        /* GP_ABI_VERSION */
  int32_t device;             /* CUDA device ordinal */
  int32_t num_objects;        /* O */
  int32_t num_templates;      /* templates per object held by THIS handle (T, or the shard size on multi-GPU),
                                 <= GP_MAX_NUM_TEMPLATES */
  int32_t num_templates_global; /* templates per object over all shards (== num_templates on one GPU) */
  int32_t template_id_stride; /* global template id = local id * stride + offset (template-interleaved shards) */
  int32_t template_id_offset;
  int32_t max_batch;          /* max detections per call */
  int32_t top_k;              /* LocalSimilarity.k (configs/model/large.yaml:37), <= 32 */
  float sim_threshold;        /* LocalSimilarity.sim_threshold (large.yaml:38) */
  float patch_threshold;      /* LocalSimilarity.patch_threshold (large.yaml:39) */
  float pixel_threshold;      /* RANSAC inlier threshold in pixels (poses.py:18) */
  int32_t patch_size;         /* 14 */
  int32_t precision;          /* GP_PRECISION_* */
  int32_t ist_bank_global;    /* 0: the IST feature bank holds this handle's templates (slots as in gp_bank_write);
                                 1: it holds ALL num_templates_global templates of every object, indexed by GLOBAL id and
                                 written with gp_bank_write_ist -- multi-GPU: descriptors are sharded, the 4x smaller IST
                                 bank is replicated so that any rank can run row a5 for any global winner */
} gp_config_t;

const char* gp_last_error(void);
int gp_abi_version(void);

/* Bytes the caller must provide for the template bank and for the per-call workspace. */
int gp_query_sizes(const gp_config_t* cfg, size_t* bank_bytes, size_t* workspace_bytes);

/* Creates a handle over caller-owned device memory (both 1024-byte aligned).  Replaces the template_data
 * PandasTensorCollection + ObjectPoseRecovery built by GigaPose.set_template_data (gigaPose.py:383-394). */
int gp_create(const gp_config_t* cfg, void* bank_mem, void* workspace_mem, gp_handle_t* out);
int gp_destroy(gp_handle_t h);

/* --- onboarding (gigaPose.py:357-398) -------------------------------------------------------------------- */

/* Writes `n` templates of object `obj` starting at local template slot `tmpl0`.
 *   feat      f32  descriptors, layout per `feat_layout`; L2-normalised `norm_passes` times on the way in
 *             (2 = raw ViT tokens: ae_net.py:69 then matching.py:229; 1 = AENet output: matching.py:229 only)
 *   mask      f32  [n, H, W] template masks; sampled nearest to 16x16 (matching.py:227)
 *   ist_feat  f32  [n, 256, 16, 16] IST backbone features (gigaPose.py:376), may be NULL if a5 is not used */
int gp_bank_write(gp_handle_t h, int obj, int tmpl0, int n, const float* feat, int feat_layout, int norm_passes,
                  const float* mask, int H, int W, const float* ist_feat, void* stream);
/* IST features only (`template_data["ist_features"]`, gigaPose.py:375-376): `n` templates of object `obj` starting at
 * IST-bank slot `tmpl0` (a GLOBAL template id when
 * cfg.ist_bank_global = 1).  ist_layout: GP_LAYOUT_CHANNEL_MAJOR [n,256,16,16] (ISTNet.forward_by_chunk's shape) or
 * GP_LAYOUT_PATCH_MAJOR [n,256 patches,256 channels] (what gp_ist_trunk_forward writes: stored as is). */
int gp_bank_write_ist(gp_handle_t h, int obj, int tmpl0, int n, const float* ist_feat, int ist_layout, void* stream);

/* Pose tables over GLOBAL template ids (ObjectPoseRecovery ctor, poses.py:13-24):
 *   K [O,3,3], M [O,Tg,3,3], poses [O,Tg,4,4], all f32. */
int gp_bank_set_poses(gp_handle_t h, const float* K, const float* M, const float* poses, void* stream);

/* IST regressor weights (ist_net.py:140-155), f32 device pointers in nn.Linear layout [out,in].  The two hidden layers
 * are packed into IEEE fp16 hi/lo planes (weights x 64, undone in the GEMM epilogue) on `stream` (tensor-core form); biases and the last layer are referenced in place
 * (the caller keeps the tensors alive).  Order: scale {w1,b1,w2,b2,w3,b3}, inplane {w1,b1,w2,b2,w3,b3}. */
int gp_set_ist_weights(gp_handle_t h, const float* const weights[12], int use_tanh, void* stream);

/* --- per batch of B detections ------------------------------------------------------------------------ */

/* Stages the query descriptors / masks / object ids (gigaPose.py:513-522; matching.py:222-225).
 *   q_feat f32 (layout/norm_passes as in gp_bank_write), q_mask f32 [B,H,W], q_obj int32 [B] 0-based. */
int gp_set_queries(gp_handle_t h, int B, const float* q_feat, int feat_layout, int norm_passes, const float* q_mask,
                   int H, int W, const int32_t* q_obj, void* stream);

typedef struct gp_candidates {   /* compact per-shard top-k records, [B,k] leading dims */
  float* score;                  /* [B,k]      per-template score (matching.py:274-278) */
  int32_t* id;                   /* [B,k]      GLOBAL template id */
  float* pts_score;              /* [B,k,256]  score_tar2src */
  uint8_t* idx;                  /* [B,k,256]  idx_tar2src */
  uint8_t* valid;                /* [B,k,256]  mask_all != 0 */
  float* rel_scale;              /* [B,k,256]   optional (NULL): IST outputs of the candidate, filled by the owning shard */
  float* rel_inplane;            /* [B,k,256,2] optional (NULL) */
} gp_candidates_t;

typedef struct gp_matches {      /* exactly the outputs of LocalSimilarity.test (matching.py:308-316) */
  int64_t* id_src;               /* [B,k] */
  float* score_src;              /* [B,k] */
  float* score_pts;              /* [B,k,256] */
  int64_t* tar_pts;              /* [B,k,256,2] (x,y) patch coordinates, -1 = invalid */
  int64_t* src_pts;              /* [B,k,256,2] */
} gp_matches_t;

/* Fused similarity search over this handle's templates + local top-k (matching.py:233-279). */
int gp_sim_candidates(gp_handle_t h, int B, const gp_candidates_t* out, void* stream);
/* Merges G candidate lists (G = 1: the local list; G > 1: after ONE all-gather over NVLink) into the global top-k
 * (score descending, then global template id ascending) and expands the winners (matching.py:279-316).
 * List g of every field starts `rank_stride_bytes * g` bytes after the field pointer (the packed all-gather
 * buffer); rank_stride_bytes = 0 means each field is a dense [G][B][k][...] array.  If the candidates carry
 * rel_scale / rel_inplane, the winners' rows are copied to out_rel_scale [B,k,256] / out_rel_inplane [B,k,256,2]. */
int gp_topk_merge(gp_handle_t h, int B, int G, const gp_candidates_t* gathered, size_t rank_stride_bytes,
                  const gp_matches_t* out, float* out_rel_scale, float* out_rel_inplane, void* stream);
/* Single-GPU convenience: gp_sim_candidates into the workspace + gp_topk_merge(G=1) == LocalSimilarity.test. */
int gp_sim_topk(gp_handle_t h, int B, const gp_matches_t* out, void* stream);

/* ISTNet.inference for all k hypotheses (ist_net.py:97-120; k-loop gigaPose.py:545-575) of the `n` detections
 * [b0, b0 + n) of the staged batch (b0 = 0, n = B: the whole batch; multi-GPU ranks each take a window).  All tensor
 * arguments are WINDOW-relative:
 *   q_ist f32 [n,256,16,16] (GP_LAYOUT_CHANNEL_MAJOR) or [n,256 patches,256] (GP_LAYOUT_PATCH_MAJOR);
 *   outputs rel_scale [n,k,256], rel_inplane [n,k,256,2] (-1000 where invalid).
 * Every template named in m->id_src must be in this handle's IST bank (all are when cfg.ist_bank_global = 1). */
int gp_ist_mlp(gp_handle_t h, int b0, int n, const float* q_ist, int ist_layout, const gp_matches_t* m, float* rel_scale,
               float* rel_inplane, void* stream);

typedef struct gp_ransac_out {   /* ObjectPoseRecovery.forward_ransac (poses.py:124-163) */
  float* M;                      /* [B,k,3,3] */
  uint8_t* failed;               /* [B,k] */
  int64_t* inlier_src_pts;       /* [B,k,256,2] */
  int64_t* inlier_tar_pts;       /* [B,k,256,2] */
  int64_t* inlier_scores;        /* [B,k,256] */
  int32_t* inlier_count;         /* [B,k] */
} gp_ransac_out_t;

/* n = number of (detection, hypothesis) pairs; src_pts/tar_pts [n,256,2] i64, rel_scale [n,256], rel_inplane
 * [n,256,2]; outputs as gp_ransac_out_t with leading dimension n.  Needs no handle (RANSAC.forward, ransac.py:108). */
int gp_ransac(int n, float pixel_threshold, int patch_size, const int64_t* src_pts, const int64_t* tar_pts,
              const float* rel_scale, const float* rel_inplane, const gp_ransac_out_t* out, void* stream);

/* ObjectPoseRecovery.forward_recovery alone (poses.py:103-122), no re-sort: q_obj int32 [B] 0-based, q_K/q_M
 * [B,3,3], id_src i64 [B,k], M [B,k,3,3], template tables K [O,3,3], M [O,T,3,3], poses [O,T,4,4] -> poses [B,k,4,4]. */
int gp_pose_recover(int B, int k, int num_templates, const int32_t* q_obj, const float* q_K, const float* q_M,
                    const int64_t* id_src, const float* M, const float* tmpl_K, const float* tmpl_M,
                    const float* tmpl_pose, float* poses, void* stream);

typedef struct gp_predictions {  /* every [B,k,...] tensor after the re-sort of gigaPose.py:588-595 + poses */
  gp_matches_t matches;
  float* rel_scale;              /* [B,k,256] */
  float* rel_inplane;            /* [B,k,256,2] */
  gp_ransac_out_t ransac;        /* inlier_count may be NULL */
  float* scores;                 /* [B,k]  inliers / 256 (gigaPose.py:588) */
  float* poses;                  /* [B,k,4,4] (poses.py:103-122) */
} gp_predictions_t;

/* scores, stable descending re-sort of the k hypotheses (skipped when sort_by_inliers = 0: the reference's
 * `sort_pred_by_inliers=False`, gigaPose.py:590) and pose lifting (gigaPose.py:588-604) for the detections
 * [b0, b0 + n) of the staged batch; every tensor argument is window-relative.
 *   q_K, q_M f32 [n,3,3] query intrinsics / crop matrices. */
int gp_sort_and_pose(gp_handle_t h, int b0, int n, int sort_by_inliers, const float* q_K, const float* q_M,
                     const gp_matches_t* m, const float* rel_scale, const float* rel_inplane, const gp_ransac_out_t* r,
                     const gp_predictions_t* out, void* stream);

/* --- row e: multi-GPU (no reference code: inference is single-GPU, configs/machine/trainer/local.yaml:4) ----------
 * One process per GPU; rank r holds the descriptor shard {tau : tau % world == r} (cfg.template_id_stride / offset). */
/* Binds an NCCL communicator (an `ncclComm_t`, e.g. torch's ProcessGroupNCCL communicator) to the handle.  The NCCL
 * entry points are resolved from the already loaded libnccl at run time (no link-time dependency).  The communicator is
 * BORROWED: it must stay alive for as long as gp_allgather / gp_topk_allgather_merge are called on this handle, and its
 * rank / size must equal cfg.template_id_offset / cfg.template_id_stride. */
int gp_comm_init(gp_handle_t h, void* nccl_comm, int rank, int world);
/* ncclAllGather of `bytes_per_rank` bytes on `stream`: recv = [world][bytes_per_rank]; send may alias its own slot. */
int gp_allgather(gp_handle_t h, const void* send, void* recv, size_t bytes_per_rank, void* stream);
/* THE collective of the search: `packed` = [world][rank_stride_bytes] holds this rank's candidate records (written by
 * gp_sim_candidates into slot `rank`); all-gathers it in place over NVLink and merges the world * k candidates per
 * detection into the global top-k (gp_topk_merge semantics).  `slot0` = field pointers of slot 0 inside `packed`. */
int gp_topk_allgather_merge(gp_handle_t h, int B, void* packed, size_t rank_stride_bytes, const gp_candidates_t* slot0,
                            const gp_matches_t* out, void* stream);

/* --- row a1: DINOv2 ViT-L/14 patch tokens (AENet.forward_by_chunk, ae_net.py:55-69; hub module un-vendored) ---- */
typedef struct gp_vit_context* gp_vit_handle_t;

/* Bytes for the packed weights (bf16 hi/lo planes) and for the activation workspace of `max_crops` crops. */
int gp_vit_query_sizes(int depth, int max_crops, size_t* weight_bytes, size_t* workspace_bytes);

/* `weights`: 4 + 14*depth f32 device pointers in upstream state-dict order --
 *   patch_embed.proj.weight [1024,3,14,14], patch_embed.proj.bias [1024], cls_token [1024],
 *   pos table [257,1024] (pos_embed already interpolated to the 16x16 grid: a weight-only computation),
 *   then per block: norm1.weight, norm1.bias, attn.qkv.weight [3072,1024], attn.qkv.bias, attn.proj.weight [1024,1024],
 *   attn.proj.bias, ls1.gamma, norm2.weight, norm2.bias, mlp.fc1.weight [4096,1024], mlp.fc1.bias,
 *   mlp.fc2.weight [1024,4096], mlp.fc2.bias, ls2.gamma.
 * GEMM weights are packed into `weight_mem` on `stream`; biases / norms / gammas / tables are referenced in place
 * (the caller keeps them alive).  precision: GP_PRECISION_FP32_SPLIT or GP_PRECISION_BF16. */
int gp_vit_create(int device, int depth, int max_crops, int precision, const float* const* weights, void* weight_mem,
                  void* workspace_mem, void* stream, gp_vit_handle_t* out);
int gp_vit_destroy(gp_vit_handle_t h);
/* img f32 [b,3,224,224] -> x_prenorm f32 [b,257,1024]: tokens after the last block, before the final norm
 * (DinoVisionTransformer.forward_features()["x_prenorm"], the tensor ae_net.py:65 slices). */
int gp_vit_forward(gp_vit_handle_t h, int b, const float* img, float* x_prenorm, void* stream);

/* AENet.forward_by_chunk's tail (ae_net.py:65-69): drops the CLS row of x_prenorm [b,257,1024] and L2-normalises every
 * patch token (F.normalize semantics) -> out f32 [b,256,1024] (patch-major; its channels-last view is the [b,1024,16,16]
 * tensor the reference module returns).  Needs no handle. */
int gp_normalize_patch_tokens(int b, const float* x_prenorm, float* out, void* stream);

/* --- rows a6 / f1: IST trunk (ResNet, resnet.py:318-381 called at ist_net.py:62-63), BatchNorm folded ------------ */
#define GP_IST_TRUNK_NUM_CONVS 21
typedef struct gp_ist_trunk_context* gp_ist_trunk_handle_t;
/* One convolution with its inference-time BatchNorm folded in (w * gamma / sqrt(var + eps), beta - mean * gamma / ...):
 *   weight f32 [cout, kh, kw, cin] (channels-last filter), bias f32 [cout] or NULL. */
typedef struct {
  const float* weight;
  const float* bias;
} gp_conv_weights_t;

int gp_ist_trunk_query_sizes(int max_crops, size_t* weight_bytes, size_t* workspace_bytes);
/* `convs`: GP_IST_TRUNK_NUM_CONVS entries in execution order -- conv1+bn1 (7x7/2, 3->128); for layer1..layer4 and block
 * 0,1: conv1+bn1 (3x3), [block 0 of layer2..4: downsample.0+downsample.1 (1x1/2),] conv2+bn2 (3x3); layer4_outconv
 * (1x1, 512->256, no bias).  Geometry is the shipped config (configs/model/ist_net/resnet.yaml: input 256, dims
 * 128/192/256/512, descriptor 256).  Weights are packed into `weight_mem` on `stream`; biases are referenced in place. */
int gp_ist_trunk_create(int device, int max_crops, int precision, const gp_conv_weights_t* convs, void* weight_mem,
                        void* workspace_mem, void* stream, gp_ist_trunk_handle_t* out);
int gp_ist_trunk_destroy(gp_ist_trunk_handle_t h);
/* crops f32 [n,3,224,224] (normalised RGB) -> feat f32 [n,256 patches,256 channels]: the [n,256,16,16] map
 * ISTNet.forward_by_chunk returns (ist_net.py:52-64), stored patch-major (the layout gp_bank_write / gp_ist_mlp keep). */
int gp_ist_trunk_forward(gp_ist_trunk_handle_t h, int n, const float* crops, float* feat, void* stream);

/* --- row f3: query pre-processing (CropResizePad.__call__, src/utils/crop.py:16-61, fused with the element-wise steps
 * of process_real, dataloader/train.py:80-123, and the CLIP normalisation, configs/data/transform.yaml:2-7) ---------- */
/* For detection i: crop xyxy_boxes[i] (i64 [n,4]; upper bounds clip to the image, negative corners clamp to 0) out of
 * images[image_index ? image_index[i] : i] (f32 [*,C,H,W]), nearest resize so that the longer box side becomes
 * target_size, centred zero padding, nearest resize to target_size x target_size -> out_images [n,C,T,T]; out_M [n,3,3]
 * (may be NULL) is the 3x3 map from image to crop pixels (the `M` GigaPose carries as tar_M / template M).
 * Optional fused element-wise steps, in the reference's order: value / in_div (255 for 8-bit data, 1 = off), x mask
 * (f32 [n,H,W] or NULL; its crop goes to out_mask [n,T,T] when that is not NULL), then after the padding
 * (value - post_sub[c]) / post_div[c] (per channel, NULL = off).  target_size >= 128 (ATen index arithmetic of large
 * outputs; the shipped configuration uses 224).  Needs no handle. */
int gp_crop_resize_pad(int n, int channels, int height, int width, int target_size, const float* images,
                       const int32_t* image_index, const int64_t* xyxy_boxes, const float* mask, float in_div,
                       const float* post_sub, const float* post_div, float* out_images, float* out_mask, float* out_M,
                       void* stream);

/* --- row f5: template renders from a CAD mesh (the Panda3D call of src/custom_megapose/call_panda3d.py:45-59 plus the
 * PNG round trip and bounding box of custom_megapose/template_dataset.py:66-119).  The full contract is the header
 * comment of gigapose_b200/csrc/render.cu.  Needs no handle. ------------------------------------------------------ */
/* Workspace bytes for up to `max_views` views of height x width: the per-sample key buffer, 8 B x 4 samples x H x W
 * per view. */
int gp_render_query_sizes(int max_views, int height, int width, size_t* workspace_bytes);
/* Renders n_views views of one triangle mesh: vertices f32 [V,3], faces i32 [F,3]; shading from vertex_color f32
 * [V,3], or texture f32 [tex_h,tex_w,3] (row 0 on top) with face_uv f32 [F,3,2], or constant_color f32 [3] (NULL =
 * white); at most one of vertex_color / texture.  poses f32 [n,4,4] object -> camera (same length unit as the
 * vertices), K f32 [3,3], z_near > 0 in that unit.  Outputs: rgba f32 [n,4,H,W], depth f32 [n,H,W] (may be NULL),
 * boxes i64 [n,4] xyxy with exclusive max ((0, 0, W, H) for an empty view).  `workspace` holds
 * gp_render_query_sizes(n_views, ...) bytes; after the call it starts with the key buffer u64 [n,H,W,4]
 * ((float bits of z) << 32 | face id, all ones = background) of this call. */
int gp_render_templates(int n_views, int height, int width, int num_vertices, const float* vertices, int num_faces,
                        const int32_t* faces, const float* vertex_color, const float* face_uv, const float* texture,
                        int tex_h, int tex_w, const float* constant_color, const float* poses, const float* K,
                        float z_near, void* workspace, float* rgba, float* depth, int64_t* boxes, void* stream);

/* --- diagnostics ----------------------------------------------------------------------------------------- */
/* number of kernels this library has launched since load (all handles); used for bench.py's `gpu_launches` */
uint64_t gp_launch_count(void);
/* times `iters` back-to-back runs of the similarity kernel alone with CUDA events on `stream`
 * (synchronises the stream); writes the average milliseconds per launch. */
int gp_time_sim_kernel(gp_handle_t h, int B, int iters, float* avg_ms, void* stream);
/* same for the 4 * depth linear layers (vit_gemm_kernel) of one ViT forward over `b` crops: average milliseconds per
 * forward's worth of linears (the residual stream is clobbered; the next gp_vit_forward rebuilds it). */
int gp_vit_time_linears(gp_vit_handle_t h, int b, int iters, float* avg_ms, void* stream);

/* diagnostics: SM-cycle stamps of CTA 0 of the last attention launch (synchronises the device); 32 int64 values:
 * [0] start, [1] Q/K landed, [2 + w] warpgroup w (0, 1) done with its query tiles; the other entries are not written. */
int gp_debug_attention_timeline(long long* stamps32);
/* same for CTA 0 of the last QKV-shaped ViT GEMM: 64 int64: [4*tile + {0: MMA start, 1: MMA done, 2: epilogue
 * start, 3: epilogue end}], [63] = kernel start. */
int gp_debug_gemm_timeline(long long* stamps64);
/* runs the first `num_convs` convolutions of the trunk and writes the last one's output as f32 NHWC */
int gp_debug_ist_trunk(gp_ist_trunk_handle_t h, int n, const float* crops, int num_convs, float* activation, void* stream);

/* test hook: runs the similarity kernel and additionally dumps the raw fp32 similarity tiles, laid out
 * [n * B + j][256 t][256 s] where j indexes the queries sorted by object id (small sizes only). */
int gp_debug_sim_tiles(gp_handle_t h, int B, float* tiles, void* stream);

/* test hook: one launch of the wgmma GEMM of the ViT / IST paths on caller-made operand planes,
 * C[M,N] = A[M,K] . W[N,K]^T (+ the fused epilogue of `mode`).  Planes are bf16 (f16 = 0) or IEEE fp16 (f16 = 1)
 * hi / lo pairs, dense row-major; every pointer is a device pointer.  Fields mirror the non-convolution part of the
 * internal GEMM parameters:
 *   mode       0 planes, 1 planes + erf-GELU, 2 x += gamma * (acc + bias), 3 patch embedding (row remap + pos table),
 *              4 QKV head-major scatter, 5 planes + ReLU, 6 planes + residual planes + ReLU, 7 fp32 rows, 8 fp32 rows + ReLU
 *   bn         output-tile width, 192 or 256 (0 = 256)
 *   swap       1: A is the 128-row operand and the outputs are written transposed, as planes [N, M]; bias is per row of A
 *   acc_scale  0 = off, else C = acc * acc_scale + bias
 *   m_dev      nullable device int32: the rows computed are min(*m_dev, M)
 * Unsupported combinations are rejected with GP_ERR_INVALID before any device is touched. */
typedef struct gp_debug_gemm {
  int32_t M, N, K, bn, passes, mode, swap, f16;
  float acc_scale;
  const uint16_t *a_hi, *a_lo;   /* [M,K] */
  const uint16_t *w_hi, *w_lo;   /* [N,K] */
  uint16_t *out_hi, *out_lo;     /* output planes (modes 0, 1, 4, 5, 6) */
  const float* bias;             /* [N] ([M] when swap) */
  const float* gamma;            /* [N] (mode 2) */
  float* x;                      /* fp32 rows (modes 2, 3, 7, 8) */
  const float* pos;              /* [tokens_per_img, N] (mode 3) */
  const uint16_t *res_hi, *res_lo;   /* residual planes, same layout as the output planes (mode 6) */
  const int32_t* m_dev;
  int32_t tokens_per_img, patches_per_img, qkv_crop_stride;
} gp_debug_gemm_t;
int gp_debug_gemm(const gp_debug_gemm_t* g, void* stream);

/* test hook: the multi-head attention kernel of the ViT alone.  qkv_hi / qkv_lo: bf16 planes in the head-major layout
 * the QKV projection writes, [3 (q|k|v)][crop_stride][16 heads][257 tokens][64]; the first b crops are attended.
 * out_hi / out_lo: bf16 planes [b * 257, 1024] (token rows, head h in columns [64 h, 64 h + 64)).  passes: 3 or 1. */
int gp_debug_attention(int b, int crop_stride, int passes, const uint16_t* qkv_hi, const uint16_t* qkv_lo, uint16_t* out_hi,
                       uint16_t* out_lo, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GIGAPOSE_B200_H_ */
