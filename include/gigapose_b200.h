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
/* Row f9: the same crop for CNOS detections whose masks are COCO run-length encodings, in place of the dense
 * `pycoco_utils.rle_to_binary_mask` masks of the reference's test loader (dataloader/test.py:238, train.py:82,107-110,
 * transform.yaml:2-7).  Outputs are those of gp_crop_resize_pad with channels = 3, the mask, in_div = 255 and the CLIP
 * mean / std, bit for bit.  images u8 [*,H,W,3] (HWC, as decoded), image_index i32 [n] (device); detection i's runs are
 * counts[offsets[i] .. offsets[i+1]) (i32, device): column-major (pixel (row, col) is run position col * H + row), the
 * first run counts zeros, runs alternate, anything past the last run is 0 and runs past H * W are cut off.  offsets
 * i64 [n+1] is HOST memory, non-decreasing from offsets[0] >= 0; ends i64 (device, offsets[n] elements) is scratch that
 * receives each detection's running sums.  out_images f32 [n,3,T,T], out_mask f32 [n,T,T], out_M f32 [n,3,3].  Two
 * launches per 256 detections.  Needs no handle. */
int gp_crop_resize_pad_rle(int n, int height, int width, int target_size, const uint8_t* images,
                           const int32_t* image_index, const int64_t* xyxy_boxes, const int32_t* counts,
                           const int64_t* offsets, int64_t* ends, float* out_images, float* out_mask, float* out_M,
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
/* Depth-only renders for the pose-error metrics (row f7; the BOP toolkit's vispy depth renderer, which the reference
 * reaches through eval_bop19_pose.py, src/scripts/eval_bop.py:16-38): the mesh, poses, K and z_near of
 * gp_render_templates, rasterised with ONE sample per pixel at the pixel centre and no shading.  Outputs: depth f32
 * [n,H,W] (0 = background), boxes i64 [n,4] of depth > 0 (xyxy, exclusive max; (0, 0, W, H) for an empty view).
 * `workspace` holds n_views * H * W * 8 bytes (one u64 depth key per pixel). */
int gp_render_depth(int n_views, int height, int width, int num_vertices, const float* vertices, int num_faces,
                    const int32_t* faces, const float* poses, const float* K, float z_near, void* workspace, float* depth,
                    int64_t* boxes, void* stream);

/* --- row f16: onboarding from real frames with known poses (BOP onboarding_static).  The full contract is the header
 * comment of gigapose_b200/csrc/onboard.cu.  Pixel centres are at integer coordinates, as gp_render_templates projects
 * with K: pixel (column c, row r) is centred at (c, r).  virtual_to_source is HOST f64 [n,3,3] (row-major), the map
 * H^-1 = K_f R_v^T K_t^-1 from a virtual pixel centre to frame pixel coordinates; a virtual pixel samples the frame at
 * (x, y) = (s0 / s2, s1 / s2), s = H^-1 (c, r, 1)^T, and lies outside it when s2 <= 0 or the nearest pixel
 * (rint(x), rint(y)) is outside [0, W) x [0, H).  Needs no handle. ----------------------------------------------------- */
#define GP_RECENTRE_MAX_SIDE 16384   /* largest side, px, of a frame's box-scan region on the virtual grid */
/* Boxes of the re-centred masks: masks u8 [n,H,W] (non-zero = object), src_boxes HOST i64 [n,4] xyxy (exclusive max)
 * holding every non-zero pixel of each mask (x2 <= x1 for an empty mask).  out_boxes i64 [n,4] (device) gets, per
 * frame, the xyxy box (exclusive max) of the virtual pixels whose nearest frame pixel is a mask pixel, on the
 * unbounded virtual grid (coordinates may be negative or beyond any image size); (0, 0, 0, 0) when there is none.
 * The scan region is the source box widened by 1 px and mapped through H; a frame whose region has a side over
 * GP_RECENTRE_MAX_SIDE, or reaches the virtual camera's horizon, is refused with GP_ERR_INVALID naming the frame. */
int gp_recentre_boxes(int n, int height, int width, const uint8_t* masks, const double* virtual_to_source,
                      const int64_t* src_boxes, int64_t* out_boxes, void* stream);
/* The 224 crops of the re-centred frames, straight from images u8 [n,H,W,3] (HWC) and masks u8 [n,H,W]: output pixel
 * -> virtual pixel with gp_crop_resize_pad's index arithmetic for boxes i64 [n,4] (device, e.g. gp_recentre_boxes'
 * output, non-empty; the box is never clipped), virtual pixel -> frame through virtual_to_source in fp64, RGB sampled
 * bilinearly (indices clamped to the frame) and the mask by nearest, then rgb / 255, x mask and the CLIP mean / std as
 * gp_crop_resize_pad_rle; 0 with mask 0 outside the frame.  Outputs out_images f32 [n,3,T,T], out_mask f32 [n,T,T] and
 * out_M f32 [n,3,3], gp_crop_resize_pad's M for the box. */
int gp_recentre_crop(int n, int height, int width, int target_size, const uint8_t* images, const uint8_t* masks,
                     const double* virtual_to_source, const int64_t* boxes, float* out_images, float* out_mask,
                     float* out_M, void* stream);

/* --- row f17: reconstruction from onboarding RGB-D frames (TSDF fusion, marching tetrahedra).  The full contract,
 * with the fp32 operation order, is the header comment of gigapose_b200/csrc/reconstruct.cu.  The grid is f32
 * [nz,ny,nx,2] of (tsdf, weight) pairs, voxel (x, y, z) centred at origin + ((x, y, z) + 0.5) * voxel in the object
 * frame (origin HOST f32 [3]).  Needs no handle. ------------------------------------------------------------------- */
#define GP_TSDF_MAX_VOXELS 134217728   /* 2^27 voxels: at most 12 triangles per cube keep counts within int32 */
/* Fuses n_frames frames into `grid` (zeroed by the caller before its first frame), in order: depth f32 [n,H,W] in the
 * unit of the poses (0 = missing), masks u8 [n,H,W] (non-zero = object), K and poses HOST f32 [n,3,3] (last row
 * 0 0 1) and [n,4,4] object -> camera; trunc = mu > 0 in the same unit. */
int gp_tsdf_fuse(int nx, int ny, int nz, const float* origin, float voxel, float trunc, int n_frames, int height,
                 int width, const float* depth, const uint8_t* masks, const float* K, const float* poses, float* grid,
                 void* stream);
/* Workspace bytes of the extraction of an nx x ny x nz grid (every side >= 2). */
int gp_tsdf_extract_query_sizes(int nx, int ny, int nz, size_t* workspace_bytes);
/* Count pass: marks the crossed edges, scans the vertex and face counts in the workspace and writes counts i64 [2]
 * (device) = (vertices, faces). */
int gp_tsdf_extract_count(int nx, int ny, int nz, const float* grid, void* workspace, int64_t* counts, void* stream);
/* Emit pass, after gp_tsdf_extract_count on the same grid and workspace: vertices f32 [V,3] in the object frame and
 * faces i32 [F,3] (V, F >= 1: the counts it wrote), both in row-major voxel order. */
int gp_tsdf_extract_emit(int nx, int ny, int nz, const float* origin, float voxel, const float* grid,
                         const void* workspace, float* vertices, int32_t* faces, void* stream);

/* --- row f7: BOP 2019 pose errors (the BOP toolkit's VSD / MSSD / MSPD that eval_bop19_pose.py computes for the
 * reference, src/scripts/eval_bop.py:16-38).  The full contract, with the fp32 operation order, is the header comment
 * of gigapose_b200/csrc/bop_eval.cu.  Needs no handle. -------------------------------------------------------------- */
#define GP_BOP_MAX_TAU 16         /* VSD misalignment tolerances per call */
#define GP_BOP_MAX_OBJECTS 256    /* objects per gp_bop_mssd_mspd call */
/* VSD (step cost, normalised by the diameter, BOP 2019 visibility) of n_pairs (estimate, ground truth) pairs.
 *   depth_test f32 [n_frames,H,W] measured depth in the model unit (0 = missing), K f32 [n_frames,3,3];
 *   est_depth f32 [n_est,H,W] / est_boxes i64 [n_est,4] and gt_depth / gt_boxes likewise (gp_render_depth outputs);
 *   per pair: frame_idx, est_idx, gt_idx i32 [n_pairs] (one render serves every pair it belongs to), diameter f32;
 *   delta > 0 and tau (HOST f32 [n_tau], 1 <= n_tau <= GP_BOP_MAX_TAU, each > 0) in the diameter-normalised unit.
 * Outputs: counts i32 [n_pairs, 2 + n_tau] = (inter, union, cost per tau), errors f32 [n_pairs, n_tau]
 * ((cost + union - inter) / union, 1 for an empty union).  A pair with an index out of range gets counts -1 and
 * errors NaN. */
int gp_bop_vsd(int n_pairs, int n_frames, int height, int width, const float* depth_test, const float* K,
               const int32_t* frame_idx, int n_est, const float* est_depth, const int64_t* est_boxes,
               const int32_t* est_idx, int n_gt, const float* gt_depth, const int64_t* gt_boxes, const int32_t* gt_idx,
               const float* diameter, float delta, int n_tau, const float* tau, int32_t* counts, float* errors,
               void* stream);
/* MSSD (model unit) and MSPD (px) of n_pairs pairs: min over the object's symmetry transforms S of max over its
 * vertices x of |P_est x - P_gt S x|, and of the distance between the two points projected with the frame's K.
 *   obj_idx i32 [n_pairs] (0-based), vertices f32 [sum V_o, 3] and syms f32 [sum S_o, 4, 4] concatenated per object,
 *   with HOST offsets vertex_offsets / sym_offsets i32 [n_objects + 1] (0 first, strictly increasing: every object has
 *   a vertex and a transform, the identity included); K f32 [n_frames,3,3], frame_idx i32 [n_pairs], pose_est /
 *   pose_gt f32 [n_pairs,4,4] object -> camera.
 * Outputs mssd, mspd f32 [n_pairs]; a pair whose object or frame index is out of range gets NaN. */
int gp_bop_mssd_mspd(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets,
                     const float* vertices, const int32_t* sym_offsets, const float* syms, int n_frames, const float* K,
                     const int32_t* frame_idx, const float* pose_est, const float* pose_gt, float* mssd, float* mspd,
                     void* stream);

/* --- row f8: BOP 2024 6D-detection score (the toolkit's eval_bop24_pose.py, which the reference's README names for
 * `test_setting: detection` runs): greedy matching with ignored ground truths and COCO average precision over MSSD /
 * MSPD.  The full contract, with the fp64 operation order, is the header comment of gigapose_b200/csrc/bop_eval.cu.
 * Needs no handle; the two calls run in stream order with no host synchronisation between them. ------------------- */
#define GP_BOP_MAX_GT_PER_GROUP 1024   /* ground truths per (image, object) group in gp_bop_match (32 x 32 flags) */
#define GP_BOP_MAX_RECALL 128          /* recall thresholds per gp_bop_average_precision call */
#define GP_BOP_MATCH_GROUP_BYTES 32    /* workspace bytes per group of gp_bop_match */
#define GP_BOP_LABEL_FP 0
#define GP_BOP_LABEL_TP 1
#define GP_BOP_LABEL_IGNORED 2
/* Greedy matching of n_groups (image, object) groups for the 2 metrics (0 = MSSD, 1 = MSPD) x n_theta thresholds.
 *   HOST tables: est_offsets / gt_offsets i32 [n_groups + 1] (0 first, non-decreasing): group g owns the estimate rows
 *   [est_offsets[g], est_offsets[g + 1]), in descending score order, and the ground truths [gt_offsets[g],
 *   gt_offsets[g + 1]) (at most GP_BOP_MAX_GT_PER_GROUP); group_obj i32 [n_groups] in [0, n_objects);
 *   thresholds f64 [n_objects, 2, n_theta], finite (1 <= n_theta <= GP_BOP_MAX_TAU).
 *   Device: mssd / mspd f32 [sum_g n_est_g * n_gt_g], each group a dense row-major [n_est, n_gt] block, the groups in
 *   order; gt_valid u8 [gt_offsets[n_groups]] (1 = valid, 0 = ignored); workspace of 8 * 2 * n_objects * n_theta +
 *   GP_BOP_MATCH_GROUP_BYTES * n_groups bytes, 8-byte aligned (the host tables are copied there in stream order
 *   before the call returns).
 * Output labels i8 [est_offsets[n_groups], 2, n_theta]: GP_BOP_LABEL_FP / _TP / _IGNORED. */
int gp_bop_match(int n_groups, int n_objects, int n_theta, const int32_t* est_offsets, const int32_t* gt_offsets,
                 const int32_t* group_obj, const double* thresholds, const float* mssd, const float* mspd,
                 const uint8_t* gt_valid, void* workspace, int8_t* labels, void* stream);
/* COCO average precision per (object, metric, threshold) from the labels of gp_bop_match.
 *   labels i8 [n_est, 2, n_theta] (device); rank i32 (device): object o's estimate rows ranked by descending score
 *   over all images at rank[rank_offsets[o] .. rank_offsets[o + 1]) (HOST offsets i32 [n_objects + 1], 0 first,
 *   non-decreasing); n_valid i32 [n_objects] (HOST, each >= 1) valid ground truths per object; recall_thresholds
 *   (HOST f64 [n_recall], finite, non-decreasing, 1 <= n_recall <= GP_BOP_MAX_RECALL).
 * Output ap f64 [n_objects, 2, n_theta] (0 for an object without estimates; NaN if a rank index is outside
 * [0, n_est)). */
int gp_bop_average_precision(int n_objects, int n_theta, int n_est, const int8_t* labels, const int32_t* rank_offsets,
                             const int32_t* rank, const int32_t* n_valid, int n_recall, const double* recall_thresholds,
                             double* ap, void* stream);

/* --- row f12: ADD, ADD-S and the 2D-projection error (LM / LM-O's ADD(-S) recall at 0.1 d, YCB-V's AUC, the 5 px
 * projection recall).  The definitions, with the fp32 / fp64 operation order, are the comment above add_kernel in
 * gigapose_b200/csrc/bop_eval.cu.  Needs no handle. ------------------------------------------------------------------ */
#define GP_BOP_ADD_CHUNK 1024          /* ground-truth vertices per partial sum of gp_bop_add */
/* ADD, ADD-S (model unit) and proj (px) of n_pairs (estimate, ground truth) pairs over every vertex of the pair's object.
 *   obj_idx i32 [n_pairs] (0-based), vertices f32 [sum V_o, 3] concatenated per object with HOST offsets
 *   vertex_offsets i32 [n_objects + 1] (0 first, strictly increasing); K f32 [n_frames,3,3], frame_idx i32 [n_pairs],
 *   pose_est / pose_gt f32 [n_pairs,4,4] object -> camera (gp_bop_mssd_mspd's tables without the symmetries);
 *   workspace of 24 * n_pairs * ceil(max_o V_o / GP_BOP_ADD_CHUNK) bytes, 8-byte aligned (the per-chunk partial sums;
 *   at most 65535 chunks).
 * Output out f64 [n_pairs, 3] = (ADD, ADD-S, proj); a pair whose object or frame index is out of range gets NaN. Two
 * launches, in stream order. */
int gp_bop_add(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets, const float* vertices,
               int n_frames, const float* K, const int32_t* frame_idx, const float* pose_est, const float* pose_gt,
               void* workspace, double* out, void* stream);

/* --- row f14: the reference's diagnostic images (vis_bop_results.py's overlays and error heat maps, plot_Kabsch's
 * retrieval panels).  The full contract, with every rounding, is the header comment of gigapose_b200/csrc/vis.cu.
 * Needs no handle; every pointer is device memory unless marked HOST. ------------------------------------------------ */
#define GP_VIS_CROP 224              /* side of the retrieval crops of gp_vis_kabsch */
#define GP_VIS_MAX_SIDE 16384        /* largest image side of gp_vis_overlay */
/* Per-vertex error of n_pairs (estimate, ground truth) pairs, in gp_bop_add's tables (obj_idx, HOST vertex_offsets,
 * vertices, pose_est, pose_gt; no frames): values f32 [out_offsets[n_pairs]], pair p's at [out_offsets[p],
 * out_offsets[p + 1]) (i64 [n_pairs + 1]; the slot length is the vertex count of the pair's object), the ADD distance
 * of each vertex, or the ADD-S distance (nearest estimated point of each ground-truth point) where symmetric u8
 * [n_pairs] is nonzero.  A pair whose object index is out of range or whose slot length differs gets NaN.  One launch. */
int gp_vis_vertex_errors(int n_pairs, int n_objects, const int32_t* obj_idx, const int32_t* vertex_offsets,
                         const float* vertices, const float* pose_est, const float* pose_gt, const uint8_t* symmetric,
                         const int64_t* out_offsets, float* values, void* stream);
/* Heat-map vertex colours of n_pairs pairs from gp_vis_vertex_errors' values, offsets and symmetric flags:
 * colors f32 [offsets[n_pairs], 3] in [0, 1] (turbo, normalised per pair over the values with max_distance appended,
 * and 0 for a symmetric pair), for gp_render_templates' vertex_color.  max_distance > 0, in the unit of the values. */
int gp_vis_heat_colors(int n_pairs, const int64_t* offsets, const uint8_t* symmetric, const float* values,
                       float max_distance, float* colors, void* stream);
/* Composites n_layers renders over one image: image u8 [H,W,3] (NULL = black) turned grey, then per layer in order
 * its RGB where its alpha > 0 and, when colors u8 [n_layers,3] is not NULL, its contour in its colour.  renders f32
 * [n_layers,4,H,W] and boxes i64 [n_layers,4] as gp_render_templates writes them.  Output out u8 [H,W,3]. */
int gp_vis_overlay(int height, int width, int n_layers, const uint8_t* image, const float* renders,
                   const int64_t* boxes, const uint8_t* colors, uint8_t* out, void* stream);
/* Retrieval panels of n (query, template, M) triples: query / tmpl f32 [n,3,224,224] normalised crops, query_mask /
 * tmpl_mask f32 [n,224,224], M f32 [n,3,3] (template crop -> query crop).  Output out u8 [n,224,224,3]: the query in
 * grey with the template warped by M pasted through its warped mask, the warped mask's edge red and the query mask's
 * edge green. */
int gp_vis_kabsch(int n, const float* query, const float* query_mask, const float* tmpl, const float* tmpl_mask,
                  const float* M, uint8_t* out, void* stream);

/* --- row f6: depth refinement of the coarse poses (MegaPose's ICPRefiner, src/megapose/inference/icp_refiner.py:134-287,
 * with a GPU point-to-plane ICP in place of OpenCV's ppf_match_3d_ICP).  The full contract is the header comment of
 * gigapose_b200/csrc/depth_icp.cu.  Needs no handle. ------------------------------------------------------------- */
#define GP_ICP_OK 0               /* refined pose accepted */
#define GP_ICP_TOO_FEW_POINTS 1   /* fewer than min_points targets or sources: T0 returned */
#define GP_ICP_DEGENERATE 2       /* singular point-to-plane system (e.g. a planar object): T0 returned */
#define GP_ICP_RESIDUAL 3         /* converged with residual > max_residual: T0 returned */
#define GP_ICP_INVALID 4          /* frame_idx outside [0, n_frames): T0 returned */
#define GP_ICP_LOST 5             /* an iteration found no pair, or kept fewer than 6: T0 returned */

/* One ICP iteration of one hypothesis (gp_icp_debug_t.trace), 456 bytes.  Written by every iteration that associates,
 * including the one that ends the refinement as LOST or DEGENERATE. */
typedef struct gp_icp_trace {
  int32_t level;                 /* L-1 .. 0 */
  int32_t iteration;             /* 0-based within the level */
  int32_t n;                     /* sources at this level, ceil(sources / 2^level) */
  int32_t found;                 /* sources with a pair */
  int32_t kept;                  /* pairs within rejection_scale x the median (0 when found = 0) */
  int32_t done;                  /* 0 step taken, 1 step taken and the level converged, 2 degenerate, 3 lost */
  uint32_t median_bits;          /* float bits of the median pair distance (+inf bits when found = 0) */
  int32_t reserved;              /* 0 */
  float Tf[12];                  /* [3,4] the fp32 correction the sources were transformed with */
  double sums[29];               /* 21 upper-triangle entries of A^T A (row by row), 6 of A^T r, sum r^2, kept */
  double xi[6];                  /* the solved step (omega L, v); 0 unless done is 0 or 1 */
  double dT[12];                 /* [3,4] the fp64 correction after the step (unchanged for done 2, 3) */
} gp_icp_trace_t;

typedef struct gp_icp_debug {    /* every field nullable; test and timing hooks */
  int32_t* counts;               /* [n_hyp,2] number of targets, sources */
  int32_t* sources;              /* [n_hyp,H*W] compacted source pixel indices (row-major), first `sources` entries */
  int32_t* assoc;                /* [n_hyp,H*W] last level-0 iteration, per level-0 source: the target pixel index of a
                                    kept pair, -2 - index of a rejected one, -1 for no pair */
  float* pose0;                  /* [n_hyp,3,4] the correction after the centroid shift, before the first iteration */
  int32_t* iterations;           /* [n_hyp,num_levels] iterations run per level (index = level); not written for
                                    levels that were not reached */
  gp_icp_trace_t* trace;         /* [n_hyp,trace_capacity] per-iteration records in order; needs trace_count */
  int32_t trace_capacity;        /* >= 1 when trace is set; records past it are counted but not written */
  int32_t* trace_count;          /* [n_hyp] records of each hypothesis (0 when it stops before iterating) */
} gp_icp_debug_t;

typedef struct gp_icp_params {
  float unit_per_m;              /* depth / translation units per metre (1000 for BOP's mm) */
  int32_t min_points;            /* n_min_points, 1000 (icp_refiner.py:178) */
  int32_t num_levels;            /* 4 (numLevels) */
  int32_t max_iters;             /* per level, 100 */
  float rejection_scale;         /* pairs farther than this x the median distance are dropped, 2.5 */
  float max_residual;            /* metres, 0.01: above it the coarse pose is kept */
  float min_step_rad;            /* a level stops after a step below both, 1e-6 rad ... */
  float min_step_m;              /* ... and 1e-6 m */
  gp_icp_debug_t debug;
} gp_icp_params_t;

/* Workspace bytes for n_frames frames and n_hyp hypotheses of height x width (17 <= sides <= 8192): 36 B per frame
 * pixel for the scene, 12 B per hypothesis pixel. */
int gp_icp_query_sizes(int n_frames, int n_hyp, int height, int width, size_t* workspace_bytes);
/* Per frame: depth f32 [n_frames,H,W] (0 = missing), K f32 [n_frames,3,3] full-image intrinsics.  Smooths the depth
 * and writes the organised target map; after the call the workspace starts with it, f32 [n_frames,H,W,6] = (x, y, z,
 * normal), z = 0 outside (0.2, 5) m. */
int gp_icp_prepare_scene(int n_frames, int height, int width, const float* depth, const float* K, float unit_per_m,
                         void* workspace, void* stream);
/* Per hypothesis, after gp_icp_prepare_scene on the same workspace: frame_idx i32 [n_hyp], masks u8 [n_hyp,H,W]
 * full-frame detection masks or NULL (threshold rule), rendered_depth f32 [n_hyp,H,W] and boxes i64 [n_hyp,4] from
 * gp_render_templates at T0 f32 [n_hyp,4,4] with the frame's K (the same K pointer as the scene).  Outputs: out_poses
 * f32 [n_hyp,4,4] (T0 bit for bit unless the status is GP_ICP_OK), out_status i32, out_residual f32 (RMS
 * point-to-plane distance, depth unit; -1 when not reached), out_fitness f32 (kept pairs / level-0 sources). */
int gp_icp_refine(int n_frames, int n_hyp, int height, int width, const int32_t* frame_idx, const uint8_t* masks,
                  const float* rendered_depth, const int64_t* boxes, const float* T0, const float* K,
                  const gp_icp_params_t* params, float* out_poses, int32_t* out_status, float* out_residual,
                  float* out_fitness, void* workspace, void* stream);
/* Row f11, masked normals (opt-in; header comment of depth_icp.cu, steps 1' and 2'): the target map of each detection
 * is smoothed within its own mask and stored over the mask's box only.  The detections are described on the HOST: */
typedef struct gp_icp_mask_set {
  int32_t n_det;                 /* 0 .. 65535 */
  const int32_t* frame;          /* [n_det] frame of each detection, in [0, n_frames) */
  const int32_t* boxes;          /* [n_det,4] mask boxes x0, y0, x1, y1, exclusive max, 0 <= x0 <= x1 <= W and
                                    0 <= y0 <= y1 <= H (x0 == x1 or y0 == y1: an empty mask); the mask reads as 0
                                    outside its box */
  const int64_t* run_offsets;    /* [n_det+1] run-length masks: detection d owns counts[run_offsets[d] ..
                                    run_offsets[d+1]), non-decreasing from >= 0; NULL for dense masks */
} gp_icp_mask_set_t;
/* Scene workspace bytes of the mask set, and box_pixels = the largest box area (the refine workspace holds
 * n_hyp * box_pixels * 12 bytes).  tiles_offset / map_offset (nullable): byte offsets in the scene workspace of the
 * mask tiles, u8, and of the maps, f32 x 6 per pixel; both hold the detections' boxes in order, each row-major
 * (box h x box w), so detection d starts at the sum of the areas of the boxes before it. */
int gp_icp_masked_query_sizes(int n_frames, int height, int width, const gp_icp_mask_set_t* set,
                              size_t* workspace_bytes, int64_t* box_pixels, size_t* tiles_offset, size_t* map_offset);
/* Writes the detection table to the start of the scene workspace and decodes every mask into a u8 box tile, from
 * either masks u8 [n_det,H,W] (dense, nonzero = in the mask) or, with set->run_offsets, counts i32 (device) in the
 * layout of gp_crop_resize_pad_rle (column-major runs, the first counting zeros; anything past the last run is 0).
 * Two launches, plus one run scan per 256 detections for run-length masks. */
int gp_icp_masked_decode(int n_frames, int height, int width, const gp_icp_mask_set_t* set, const uint8_t* masks,
                         const int32_t* counts, void* workspace, void* stream);
/* After gp_icp_masked_decode on the same workspace and mask set: depth f32 [n_frames,H,W], K f32 [n_frames,3,3].
 * Writes each detection's map, f32 [box h, box w, 6] = (x, y, z, normal) with normals of the depth smoothed within its
 * mask, in box order after the tiles.  Three launches. */
int gp_icp_prepare_masked_scene(int n_frames, int height, int width, const gp_icp_mask_set_t* set, const float* depth,
                                const float* K, float unit_per_m, void* workspace, void* stream);
/* gp_icp_refine with hypothesis i refined against the map and mask of detection det_idx[i] (i32 [n_hyp], device; out
 * of range: GP_ICP_INVALID); K is the scene's, the other arguments and outputs are gp_icp_refine's.  scene_workspace
 * is the prepared scene; workspace holds n_hyp * box_pixels * 12 bytes of scratch. */
int gp_icp_refine_masked(int n_frames, int height, int width, const gp_icp_mask_set_t* set, int n_hyp,
                         const int32_t* det_idx, const float* rendered_depth, const int64_t* boxes, const float* T0,
                         const float* K, const gp_icp_params_t* params, float* out_poses, int32_t* out_status,
                         float* out_residual, float* out_fitness, const void* scene_workspace, void* workspace,
                         void* stream);
/* test hook: the exact median select of gp_icp_refine alone, in one 256-thread CTA.  bits u32 [n] (float bits of
 * non-negative distances; 0x7f800000 = no pair, skipped) -> out u32 [2]: m = the entries that are not 0x7f800000, and
 * the bits of the element of rank `rank` (0-based, ascending) among them, or 0x7f800000 when rank >= m.  n >= 1,
 * 0 <= rank < n; arguments are checked before any device work. */
int gp_debug_icp_select(const uint32_t* bits, int n, int rank, uint32_t* out, void* stream);

/* --- row f13: depth refinement with MegaPose's TeaserppRefiner (src/megapose/inference/teaserpp_refiner.py:165-291):
 * pixel-aligned correspondences, farthest-point sampled, an exact maximum clique of the pairwise-consistency graph,
 * GNC-TLS rotation and voted translation.  The full contract is the header comment of
 * gigapose_b200/csrc/depth_teaser.cu.  Needs no handle. --------------------------------------------------------- */
#define GP_TEASER_MAX_POINTS 1024
#define GP_TEASER_OK 0                 /* solved and at least min_inliers inliers: [R|t] T0 written */
#define GP_TEASER_TOO_FEW_POINTS 1     /* fewer than min_points masked pixels: T0 returned */
#define GP_TEASER_CLIQUE_TOO_SMALL 2   /* maximum clique of fewer than 3 correspondences: T0 returned */
#define GP_TEASER_CLIQUE_BUDGET 3      /* the clique search visited clique_budget nodes without finishing: T0 returned */
#define GP_TEASER_TOO_FEW_INLIERS 4    /* fewer than min_inliers samples within noise_bound after the solve: T0 */
#define GP_TEASER_INVALID 5            /* frame_idx outside [0, n_frames): T0 returned */

/* One GNC-TLS iteration of one hypothesis (gp_teaser_debug_t.gnc), 112 bytes. */
typedef struct gp_teaser_gnc {
  int32_t iteration;             /* 0-based */
  int32_t members;               /* clique size m = number of chain TIMs */
  int32_t stopped;               /* 1: the mu initialisation ended the loop (mu not > 0 or not finite) */
  int32_t reserved;              /* 0 */
  double mu;                     /* the mu of this iteration's thresholds (at iteration 0 the initialised value) */
  double cost;                   /* sum of the updated weights x residuals (0 when stopped) */
  double max_residual;           /* largest squared TIM residual under R */
  double R[9];                   /* the rotation solved with this iteration's weights, row-major */
} gp_teaser_gnc_t;

typedef struct gp_teaser_debug { /* every field nullable; test and timing hooks */
  int32_t* counts;               /* [n_hyp,4] masked points N (-1: invalid frame), samples M, clique-search nodes,
                                    GNC iterations */
  float* points;                 /* [n_hyp,H*W,6] compacted (source xyz, target xyz), first N rows */
  int32_t* samples;              /* [n_hyp,n_points] sampled point indices, first M entries */
  uint32_t* adjacency;           /* [n_hyp,n_points,32] consistency graph rows of the samples, first M rows */
  int32_t* clique;               /* [n_hyp,n_points] clique members (sample indices) ascending, -1 after the last */
  gp_teaser_gnc_t* gnc;          /* [n_hyp,gnc_capacity] per-iteration records; iterations past it are not written */
  double* gnc_weights;           /* [n_hyp,gnc_capacity,n_points] the weights each iteration's rotation used; needs gnc */
  int32_t gnc_capacity;
  int32_t stop_after;            /* timing: 0 runs everything; 1 compaction, 2 + sampling, 3 + graph and order, 4 + clique
                                    only, with status -1 and T0 written where a hypothesis got that far */
  double* transform;             /* [n_hyp,12] the solved R (row-major) and t, where the solve ran */
} gp_teaser_debug_t;

typedef struct gp_teaser_params {
  float unit_per_m;              /* depth / translation units per metre (1000 for BOP's mm) */
  int32_t min_points;            /* n_min_points, 100 (teaserpp_refiner.py:172) */
  int32_t n_points;              /* samples, 1000 (n_points); 3 .. GP_TEASER_MAX_POINTS */
  float noise_bound;             /* metres, 0.01 */
  float cbar2;                   /* 1 */
  int32_t min_inliers;           /* 50 */
  float gnc_factor;              /* rotation_gnc_factor, 1.4 */
  int32_t gnc_max_iters;         /* rotation_max_iterations, 100 */
  double gnc_cost_threshold;     /* rotation_cost_threshold in m^2, 1e-12 (scaled by unit_per_m^2) */
  int64_t clique_budget;         /* clique-search nodes before GP_TEASER_CLIQUE_BUDGET (the reference has no limit) */
  gp_teaser_debug_t debug;
} gp_teaser_params_t;

/* Workspace bytes for n_hyp hypotheses of height x width: 28 B per hypothesis pixel plus 260 KiB per hypothesis. */
int gp_teaser_query_sizes(int n_hyp, int height, int width, size_t* workspace_bytes);
/* Per hypothesis: frame_idx i32 [n_hyp], depth f32 [n_frames,H,W] measured (not > 0 = missing), rendered_depth f32
 * [n_hyp,H,W] and boxes i64 [n_hyp,4] from gp_render_templates at T0 f32 [n_hyp,4,4] with the frame's K f32
 * [n_frames,3,3].  Outputs: out_poses f32 [n_hyp,4,4] (T0 bit for bit unless the status is GP_TEASER_OK),
 * out_status i32, out_inliers i32 (0 where the solve did not run), out_clique i32 (the clique size, 0 where the search
 * did not run; the best found so far on GP_TEASER_CLIQUE_BUDGET).  Three launches. */
int gp_teaser_refine(int n_frames, int n_hyp, int height, int width, const int32_t* frame_idx, const float* depth,
                     const float* rendered_depth, const int64_t* boxes, const float* T0, const float* K,
                     const gp_teaser_params_t* params, float* out_poses, int32_t* out_status, int32_t* out_inliers,
                     int32_t* out_clique, void* workspace, void* stream);

/* --- row f10: depth-consistency score of the hypotheses of each detection, and the best one.  The full contract is the
 * header comment of gigapose_b200/csrc/depth_score.cu.  Needs no handle. ------------------------------------------ */
/* frame_idx i32 [n_det]; depth f32 [n_frames,H,W] measured (not > 0 = missing); rendered f32 [n_det*n_hyp,H,W] the
 * render of each pose (0 = background) and boxes i64 [n_det*n_hyp,4] as gp_render_templates writes them, hypothesis j
 * of detection d at row d * n_hyp + j; tolerance >= 0 in the depth unit.  Outputs: counts i32 [n_det*n_hyp,4] =
 * (consistent, behind, front, missing) over the rendered pixels, score f32 [n_det*n_hyp] = consistent / (consistent +
 * behind + front) (0 for an empty denominator), best i32 [n_det] = the hypothesis with the largest score, the lowest
 * index on a tie.  A detection whose frame index is out of range gets counts -1, scores NaN and best -1. */
int gp_depth_score(int n_frames, int n_det, int n_hyp, int height, int width, const int32_t* frame_idx,
                   const float* depth, const float* rendered, const int64_t* boxes, float tolerance, int32_t* counts,
                   float* score, int32_t* best, void* stream);

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
/* same for CTA 0 of the last gp_debug_gemm launch with `stamp` set: 128 int64, for the CTA's first 15 tiles
 * [4*tile + {0: MMA start, 1: MMA done, 2: epilogue start, 3: epilogue end}] and [64 + tile] = the tile's first
 * k-block has landed in shared memory; [63] = kernel start.  Other entries are not written. */
int gp_debug_gemm_timeline(long long* stamps128);
/* runs the first `num_convs` convolutions of the trunk (0 <= num_convs < GP_IST_TRUNK_NUM_CONVS) and writes the last
 * one's output planes, merged (hi + lo), as f32 NHWC [n, h, w, c].  num_convs = 0 writes the stem's input instead: the
 * bilinear-resized crops, merged, as f32 [n, 262, 264, 4] -- pixel (y, x) of the 256 x 256 crop at row y + 3, column
 * x + 4, channels 0-2; the 3-row / 4-column border and channel 3 are zero (the stem convolution's padding). */
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
 *   stamp      1: CTA 0 records the cycle timeline read by gp_debug_gemm_timeline
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
  int32_t stamp;
} gp_debug_gemm_t;
int gp_debug_gemm(const gp_debug_gemm_t* g, void* stream);

/* test hook: the multi-head attention kernel of the ViT alone.  qkv_hi / qkv_lo: bf16 planes in the head-major layout
 * the QKV projection writes, [3 (q|k|v)][crop_stride][16 heads][257 tokens][64]; the first b crops are attended.
 * out_hi / out_lo: bf16 planes [b * 257, 1024] (token rows, head h in columns [64 h, 64 h + 64)).  passes: 3 or 1. */
int gp_debug_attention(int b, int crop_stride, int passes, const uint16_t* qkv_hi, const uint16_t* qkv_lo, uint16_t* out_hi,
                       uint16_t* out_lo, void* stream);

/* test hook: the LayerNorm kernel of the ViT alone, with the eps gp_vit_forward uses (1e-6).  x f32 [M, 1024] rows,
 * w / b f32 [1024]; out_hi / out_lo: bf16 planes [M, 1024] of (x - mean) / sqrt(var + eps) * w + b.  M >= 1. */
int gp_debug_layernorm(int M, const float* x, const float* w, const float* b, uint16_t* out_hi, uint16_t* out_lo,
                       void* stream);

#ifdef __cplusplus
}
#endif
#endif /* GIGAPOSE_B200_H_ */
