"""`GigaPose` -- drop-in for the inference half of `src/models/gigaPose.py` (Hydra target
`src.models.gigaPose.GigaPose`, configs/model/large.yaml:1).  Same constructor, same attributes `test.py` sets
after construction (`template_datasets`, `test_dataset_name`, `max_num_dets_per_forward`, `run_id`, `log_interval`,
test.py:67-74), same Lightning hooks (`test_step`, `on_test_epoch_end`), same per-image `.npz` output
(gigaPose.py:439-448).

What changed underneath (SURVEY.md §3.1): the template bank lives in kernel-native layout inside an
`Engine` (no per-detection 830 MB gathers, gigaPose.py:520-521,552), the IST backbone runs once per batch
instead of k=5 times (gigaPose.py:553), and rows a3-a9 are five kernel launches with no host synchronisation in
between.  Training / validation (`gigaPose.py:79-355`) is out of scope for this package.
"""
import os
import os.path as osp

import numpy as np
import pandas as pd
import torch

import src.megapose.utils.tensor_collection as tc
from src.models._lightning import LightningModule
from src.models.poses import ObjectPoseRecovery
from src.utils.logging import get_logger

logger = get_logger(__name__)


class _HostResult:
    """Pinned host copies of one batch's `pred_poses` / `scores`, valid after `result()` returned."""

    def __init__(self, poses, scores, done):
        self._poses, self._scores, self._done = poses, scores, done

    def result(self):
        self._done.synchronize()
        return self._poses, self._scores


RENDERS_NOT_KEPT = "renders not kept"      # GigaPose.template_views entry of a bank built by onboard_templates


class CropViews:
    """GigaPose.template_views entry of a bank built by onboard_images: `views(o, ids)` returns the template crops
    (rgb [n,3,224,224], mask [n,224,224]) themselves rather than renders to crop."""

    def __init__(self, views):
        self.views = views


def object_indices(infos, num_objects: int) -> np.ndarray:
    """0-based object indices from the `label` column (1-based ids as strings, gigaPose.py:514-520).  The reference
    indexes `template_data.ae_features[label - 1]`: label 0 silently wraps to the last object and label > O raises;
    here both raise (the kernels index the resident bank with these values)."""
    idx = np.asarray(infos.label).astype(np.int64) - 1
    if idx.size and (idx.min() < 0 or idx.max() >= num_objects):
        bad = sorted(set((idx[(idx < 0) | (idx >= num_objects)] + 1).tolist()))
        raise IndexError(f"object labels {bad} outside [1, {num_objects}] (the onboarded bank has {num_objects} objects)")
    return idx


def weights_fingerprint(*modules) -> str:
    """Content hash of every parameter / buffer of the encoders (two moments per tensor, one device->host copy):
    the on-disk bank cache is only valid for the weights it was encoded with (ADVICE r1)."""
    import hashlib
    h = hashlib.sha1()
    sums = []
    for m in modules:
        for name, t in list(m.named_parameters()) + list(m.named_buffers()):
            h.update(name.encode())
            h.update(str(tuple(t.shape)).encode())
            if t.numel() and t.is_floating_point():
                d = t.detach().double()
                sums.append(torch.stack([d.sum(), d.abs().sum()]))
    if sums:
        h.update(torch.stack(sums).cpu().numpy().tobytes())
    return h.hexdigest()[:16]


class _BankBuilder:
    """Row f2: streams the template crops of consecutive objects through both encoders in FULL chunks (the reference, and
    round 1 here, encoded one object at a time: 162 crops = 64 + 64 + 34, i.e. a ragged last ViT pass per object) and
    writes descriptors / sampled masks / IST features straight into the engine's bank in the kernel-native layout
    (the trunk's patch-major output is stored as is: no transposes on the way)."""

    def __init__(self, model, eng, chunk=64):
        self.model, self.eng, self.chunk = model, eng, chunk
        self.rgb, self.mask, self.segs, self.count, self.crops = [], [], [], 0, 0

    def add(self, obj, rgb, mask):
        T, t0 = rgb.shape[0], 0
        while t0 < T:
            take = min(self.chunk - self.count, T - t0)
            self.rgb.append(rgb[t0:t0 + take])
            self.mask.append(mask[t0:t0 + take])
            self.segs.append((obj, t0, take))
            self.count += take
            t0 += take
            if self.count == self.chunk:
                self.flush()

    def flush(self):
        if not self.count:
            return
        rgb = torch.cat(self.rgb) if len(self.rgb) > 1 else self.rgb[0]
        mask = torch.cat(self.mask) if len(self.mask) > 1 else self.mask[0]
        tokens = self.model.ae_net.raw_tokens(rgb)                    # [n,257,1024] x_prenorm; CLS drop + both normalisations in-kernel
        ist = self.model.ist_net.forward_by_chunk(rgb)                # [n,256,16,16] (channels-last view of patch-major)
        off = 0
        for obj, t0, n in self.segs:
            self.eng.bank_write(obj, t0, tokens[off:off + n], mask[off:off + n], ist_feat=ist[off:off + n],
                                norm_passes=2)                        # ae_net.py:69 + matching.py:229
            off += n
        self.crops += self.count
        self.rgb, self.mask, self.segs, self.count = [], [], [], 0


class GigaPose(LightningModule):
    def __init__(self, model_name, ae_net, ist_net, training_loss, testing_metric, optim_config, log_interval, log_dir,
                 max_num_dets_per_forward=None, test_setting="localization", **kwargs):
        super().__init__()
        self.model_name = model_name
        self.ae_net = ae_net
        self.ist_net = ist_net
        self.training_loss = training_loss
        self.testing_metric = testing_metric
        self.max_num_dets_per_forward = max_num_dets_per_forward   # memory knob of the reference; not needed here
        self.test_setting = test_setting
        self.log_interval = log_interval
        self.log_dir = log_dir
        os.makedirs(osp.join(self.log_dir, "predictions"), exist_ok=True)
        self.optim_config = optim_config
        self.optim_name = "AdamW"
        # testing state
        self.template_datas = {}
        self.pose_recovery = {}
        self.engines = {}
        self.run_id = None
        self.template_datasets = None
        self.test_dataset_name = None
        self.max_dets_per_call = int(kwargs.get("max_dets_per_call", 128))
        self.bank_cache_dir = kwargs.get("bank_cache_dir", None)         # row f2: on-disk cache of the encoded bank
        self.last_times = {}
        self.profile_stages = False          # bench.py --stage-times: CUDA events between the stages of retrieve()
        self.stage_ms = {}
        # opt-in: replay the per-batch launch sequence (~250 kernels) as one CUDA graph per batch size
        self.use_cuda_graph = bool(kwargs.get("cuda_graph", False))
        self._graphs = {}
        # row f14: how `template_crops` gets each dataset's template crops back: a view renderer after onboard_meshes,
        # a CropViews after onboard_images, RENDERS_NOT_KEPT after onboard_templates, no entry after set_template_data
        # (read from template_datasets)
        self.template_views = {}
        self.onboarding_views = {}           # row f16: frames chosen per template view by onboard_images

    # ------------------------------------------------------------------ out of scope: training
    def training_step(self, *a, **k):
        raise NotImplementedError("gigapose_b200 covers the inference hot path only (train.py is out of scope)")

    validation_step = training_step
    configure_optimizers = training_step

    # ------------------------------------------------------------------ onboarding (gigaPose.py:357-398)
    @torch.no_grad()
    def set_template_data(self, dataset_name):
        from gigapose_b200.engine import Engine
        dataset = self.template_datasets[dataset_name]
        device = self.device
        n_obj = len(dataset)
        first = dataset[0]
        T = first.rgb.shape[0]
        k = self.testing_metric.k
        eng = Engine(n_obj, T, self.max_dets_per_call, device=device, k=k,
                     sim_threshold=self.testing_metric.sim_threshold, patch_threshold=self.testing_metric.patch_threshold,
                     precision=getattr(self.testing_metric, "precision", "fp32_split"))
        Ks, Ms, poses = [], [], []
        start = torch.cuda.Event(enable_timing=True)
        stop = torch.cuda.Event(enable_timing=True)
        start.record()
        # row f2: with `bank_cache_dir` set, the encoded bank is read back from disk instead of re-running both
        # backbones over all O x T template crops (the cache is only valid for the weights it was written with)
        cache = None
        if getattr(self, "bank_cache_dir", None):
            os.makedirs(self.bank_cache_dir, exist_ok=True)
            # the file is bound to the encoder weights and to the template content (first object's crops + masks): a
            # cache written with another checkpoint, or stale renders under the same dataset name, is not loaded
            content = torch.stack([first.rgb.double().sum(), first.mask.double().sum()]).cpu().numpy().tobytes().hex()[:16]
            eng.fingerprint = weights_fingerprint(self.ae_net, self.ist_net.backbone) + "-" + content + \
                f"-{tuple(first.mask.shape[-2:])}"
            cache = osp.join(self.bank_cache_dir, f"{dataset_name}_{n_obj}x{T}_{eng.precision}.gpbank")
        cached = False
        if cache is not None and osp.exists(cache):
            from gigapose_b200._lib import GigaPoseNativeError
            try:
                eng.load_bank(cache)
                cached = True
            except GigaPoseNativeError as e:           # other weights / shape / ABI: rebuild and overwrite
                logger.info(f"bank cache {cache} not usable ({e}); re-encoding the templates")
        builder = _BankBuilder(self, eng)
        for idx in range(n_obj):
            data = first if idx == 0 else dataset[idx]
            if not cached:
                builder.add(idx, data.rgb.to(device, non_blocking=True), data.mask.to(device, non_blocking=True))
            Ks.append(data.K.to(device))
            Ms.append(data.M.to(device))
            poses.append(data.poses.to(device))
        builder.flush()
        K, M, P = torch.stack(Ks).float(), torch.stack(Ms).float(), torch.stack(poses).float()
        eng.set_poses(K, M, P)
        eng.set_ist_weights(self.ist_net.regressor)
        if cache is not None and not cached:
            eng.save_bank(cache)
        stop.record()
        stop.synchronize()
        self.engines[dataset_name] = eng
        self.template_datas[dataset_name] = tc.PandasTensorCollection(infos=pd.DataFrame(), K=K, M=M, poses=P)
        self.pose_recovery[dataset_name] = ObjectPoseRecovery(template_K=K, template_Ms=M, template_poses=P)
        self.template_views.pop(dataset_name, None)                 # template_crops reads template_datasets
        self.onboarding_s_per_object = start.elapsed_time(stop) / 1e3 / n_obj
        logger.info(f"Init {dataset_name} done! Avg time={self.onboarding_s_per_object:.3f} s/object")

    @torch.no_grad()
    def onboard_templates(self, dataset_name, rgba, boxes, K, poses):
        """Row f2, from raw renders: the whole `TemplateSet.__getitem__` + `set_template_data` sequence
        (dataloader/template.py:55-81 -> gigaPose.py:357-398) on the GPU for all objects at once.

        rgba  [O,T,4,H,W] float in [0,1] (rendered RGB + alpha; uint8 / 255 is fine) or a list of O such tensors,
        boxes [O,T,4] xyxy template boxes, K [3,3] or [O,3,3] template intrinsics, poses [O,T,4,4].
        Crop + resize + pad (`CropResizePad`, utils/crop.py:16-61) and the CLIP normalisation of the RGB channels
        (template.py:71-73) run as one gather kernel per object (`gp_crop_resize_pad`); the crops then stream through the
        ViT / IST encoders in full 64-crop chunks across object boundaries into the bank."""
        # the caller's renders are not kept: they can be [O,T,4,H,W] f32, gigabytes, and are freed with the caller's copy
        return self._onboard(dataset_name, len(rgba), rgba[0].shape[0],
                             lambda o: (rgba[o].to(self.device, non_blocking=True).float(), boxes[o]), K, poses,
                             RENDERS_NOT_KEPT)

    @torch.no_grad()
    def onboard_meshes(self, dataset_name, meshes, poses, K=None):
        """Row f5: onboarding straight from CAD meshes, with no renderer outside this library.  Each object's template
        views are rendered on the GPU (`gigapose_b200.render.render_templates`, 640 x 480, the reference's Panda3D
        template set-up of call_panda3d.py:45-59) and stream through the same crop -> encoders -> bank sequence as
        `onboard_templates`; only one object's renders are resident at a time.

        meshes  list of PLY paths or `read_ply` dicts (vertices in the unit of the pose translations, mm for BOP),
        poses   [T,4,4] (the same views for every object) or [O,T,4,4] object -> camera,
        K       [3,3] template intrinsics, default the reference's (`render.TEMPLATE_K`)."""
        from gigapose_b200.render import TEMPLATE_K, read_ply, render_templates
        K = TEMPLATE_K if K is None else K
        n_obj = len(meshes)
        poses = torch.as_tensor(poses, dtype=torch.float32)
        poses = poses.expand(n_obj, *poses.shape[-3:]) if poses.dim() == 3 else poses

        def views(o, ids):
            mesh = read_ply(meshes[o]) if isinstance(meshes[o], (str, os.PathLike)) else meshes[o]
            r = render_templates(mesh, poses[o][ids].to(self.device), K, device=self.device)
            return r["rgba"], r["boxes"]

        return self._onboard(dataset_name, n_obj, poses.shape[1], lambda o: views(o, slice(None)), K, poses, views)

    @torch.no_grad()
    def onboard_images(self, dataset_name, frames, template_poses):
        """Row f16: onboarding from real frames with known poses, for objects without a CAD model (BOP's
        onboarding_static sequences).  frames: one entry per object (label 1 first), each a
        `gigapose_b200.onboarding.Frames` or a dict(images, masks, K [n,3,3], poses [n,4,4] object -> camera) with the
        images as paths or u8 [H,W,3] and the masks as paths or [H,W] (non-zero = object); template_poses [T,4,4] the
        viewpoints to cover.  For every template viewpoint the frame seen from the nearest direction is chosen
        (`onboarding.select_frames`), re-centred on the object origin by a virtual camera with the template
        intrinsics (`onboarding.recentre`) and cropped on the GPU (gp_recentre_boxes, gp_recentre_crop); the crops go
        through the encoders into the bank as `onboard_templates`' do, with K = `render.TEMPLATE_K` and the virtual
        poses.  `onboarding_views[dataset_name]` keeps the chosen frame ids and the angular gaps (degrees) per
        object."""
        import concurrent.futures

        from gigapose_b200 import onboarding
        from gigapose_b200.render import TEMPLATE_K
        objs = [f if isinstance(f, onboarding.Frames) else onboarding.Frames(f["images"], f["masks"], f["K"], f["poses"])
                for f in frames]
        tpl = np.asarray(template_poses.cpu() if torch.is_tensor(template_poses) else template_poses, np.float64)
        tpl = tpl.reshape(-1, 4, 4)
        n_obj, T = len(objs), tpl.shape[0]
        pool = concurrent.futures.ThreadPoolExecutor(onboarding.DECODE_THREADS)
        chosen, poses = [], torch.empty(n_obj, T, 4, 4)
        try:
            def crops(o):
                ids, gaps = onboarding.select_frames(objs[o], tpl, pool)
                r = onboarding.recentre_frames(objs[o], ids, self.device, pool)
                poses[o] = torch.as_tensor(r["poses"], dtype=torch.float32)
                chosen.append((ids, gaps))
                logger.info(f"{dataset_name} object {o + 1}: {len(np.unique(ids))} of {len(objs[o])} frames for {T} "
                            f"views, largest gap {gaps.max():.1f} deg")
                return r["images"], r["mask"], r["M"]

            def views(o, ids):
                r = onboarding.recentre_frames(objs[o], np.asarray(chosen[o][0])[np.asarray(ids)], self.device)
                return r["images"].contiguous(), r["mask"].contiguous()

            eng = self._onboard_crops(dataset_name, n_obj, T, crops, TEMPLATE_K, poses, CropViews(views))
        finally:
            pool.shutdown(wait=True)
        self.onboarding_views[dataset_name] = dict(frame_ids=[c[0] for c in chosen], gap_deg=[c[1] for c in chosen])
        logger.info(f"{dataset_name}: largest angular gap to a template view {max(c[1].max() for c in chosen):.1f} deg")
        return eng

    def _onboard(self, dataset_name, n_obj, T, produce, K, poses, views):
        """The body of the render-based onboarding entry points: `produce(o)` -> (rgba [T,4,H,W] f32 on the device,
        boxes [T,4]) cropped by `crop_resize_pad`; `views(o, ids)` the same for the views `ids` only, kept for
        `template_crops` (or RENDERS_NOT_KEPT)."""
        from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad

        def crops(o):
            rgba, boxes = produce(o)
            crop = crop_resize_pad(torch.as_tensor(boxes), rgba, 224,
                                   mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,))      # alpha channel passes through
            return crop["images"][:, :3], crop["images"][:, 3], crop["M"]

        return self._onboard_crops(dataset_name, n_obj, T, crops, K, poses, views)

    def _onboard_crops(self, dataset_name, n_obj, T, crops, K, poses, views):
        """The body of every onboarding entry point: `crops(o)` -> (rgb [T,3,224,224] normalised, mask [T,224,224],
        M [T,3,3]) on the device, streamed through both encoders into a new bank with K and poses."""
        from gigapose_b200.engine import Engine
        device = self.device
        metric = self.testing_metric
        eng = Engine(n_obj, T, self.max_dets_per_call, device=device, k=metric.k, sim_threshold=metric.sim_threshold,
                     patch_threshold=metric.patch_threshold, precision=getattr(metric, "precision", "fp32_split"))
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        builder = _BankBuilder(self, eng)
        Ms = []
        for o in range(n_obj):
            rgb, mask, M = crops(o)
            builder.add(o, rgb, mask)
            Ms.append(M)
        builder.flush()
        K = torch.as_tensor(K, dtype=torch.float32, device=device)
        K = K.expand(n_obj, 3, 3).contiguous() if K.dim() == 2 else K
        M = torch.stack(Ms).float()
        P = torch.as_tensor(poses, dtype=torch.float32, device=device)
        eng.set_poses(K, M, P)
        eng.set_ist_weights(self.ist_net.regressor)
        stop.record()
        stop.synchronize()
        self.engines[dataset_name] = eng
        self.template_datas[dataset_name] = tc.PandasTensorCollection(infos=pd.DataFrame(), K=K, M=M, poses=P)
        self.pose_recovery[dataset_name] = ObjectPoseRecovery(template_K=K, template_Ms=M, template_poses=P)
        self.template_views[dataset_name] = views
        self.onboarding_s_per_object = start.elapsed_time(stop) / 1e3 / n_obj
        logger.info(f"Onboarded {dataset_name}: {n_obj} objects x {T} templates, {self.onboarding_s_per_object:.3f} s/object")
        return eng

    # ------------------------------------------------------------------ row f14: retrieval panels (gigaPose.py:451-479)
    @torch.no_grad()
    def template_crops(self, dataset_name, obj, ids):
        """The normalised template crops f32 [n,3,224,224] and masks f32 [n,224,224] of views `ids` of object index
        `obj` (0-based) as the bank was built from them: read from `template_datasets` after `set_template_data`, and
        re-rendered and re-cropped (the same `crop_resize_pad`) after `onboard_meshes`, and re-decoded and re-centred
        after `onboard_images`.  After `onboard_templates` the caller's renders are not kept, so there is nothing to read them from: that raises ValueError."""
        from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad
        ids = torch.as_tensor(np.asarray(ids, np.int64))
        views = self.template_views.get(dataset_name)
        if views is RENDERS_NOT_KEPT:
            raise ValueError(f"{dataset_name} was onboarded from caller renders (onboard_templates), which are not kept: "
                             "its template crops are not available; onboard it with onboard_meshes or set_template_data")
        if views is None:
            data = self.template_datasets[dataset_name][obj]
            return data.rgb[ids].to(self.device).float(), data.mask[ids].to(self.device).float()
        if isinstance(views, CropViews):
            return views.views(obj, ids)
        rgba, boxes = views(obj, ids)
        crop = crop_resize_pad(torch.as_tensor(boxes), rgba, 224, mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,))
        return crop["images"][:, :3].contiguous(), crop["images"][:, 3].contiguous()

    @torch.no_grad()
    def vis_retrieval(self, dataset_name, batch, predictions, selected=None):
        """The reference's retrieval panels (plot_Kabsch, src/libVis/torch.py) for the k retrieved templates of each
        detection: the template warped by its predicted affine M onto the grey query crop, the warped mask's edge red
        and the query mask's edge green (`gigapose_b200.vis.kabsch`; the keypoint panel is not drawn).  `predictions`
        is what `eval_retrieval` returns for `batch`, `selected` its batch rows (default: all of them).
        -> f32 [k * B, 3, 224, 224] in [0, 1], rank-major as the reference concatenates them."""
        from gigapose_b200.vis import kabsch
        eng = self.engines[dataset_name]
        obj = object_indices(predictions.infos, eng.O)
        B, k = predictions.id_src.shape[:2]
        rows = torch.as_tensor(np.arange(B) if selected is None else np.asarray(selected, np.int64), device=eng.device)
        tar_img, tar_mask = batch.tar_img.to(eng.device)[rows], batch.tar_mask.to(eng.device)[rows].float()
        ids = predictions.id_src.long().cpu().numpy()
        src_img = torch.empty(B, k, 3, 224, 224, device=eng.device)
        src_mask = torch.empty(B, k, 224, 224, device=eng.device)
        for o in np.unique(obj):
            b = np.nonzero(obj == o)[0]
            views, inv = np.unique(ids[b].reshape(-1), return_inverse=True)
            rgb, mask = self.template_crops(dataset_name, int(o), views)
            src_img[b] = rgb[inv].reshape(len(b), k, 3, 224, 224)
            src_mask[b] = mask[inv].reshape(len(b), k, 224, 224)
        M = predictions.M.float()
        q = tar_img.float().unsqueeze(1).expand(B, k, 3, 224, 224).transpose(0, 1).reshape(k * B, 3, 224, 224)
        qm = tar_mask.unsqueeze(1).expand(B, k, 224, 224).transpose(0, 1).reshape(k * B, 224, 224)
        panels = kabsch(q.contiguous(), qm.contiguous(), src_img.transpose(0, 1).reshape(k * B, 3, 224, 224).contiguous(),
                        src_mask.transpose(0, 1).reshape(k * B, 224, 224).contiguous(),
                        M.transpose(0, 1).reshape(k * B, 3, 3).contiguous())
        return panels.permute(0, 3, 1, 2).float() / 255.0

    # ------------------------------------------------------------------ row f6: depth refinement (icp_refiner.py:134-287)
    def attach_meshes(self, dataset_name, meshes):
        """Uploads the CAD meshes of `dataset_name` once for `refine_depth`: PLY paths or `read_ply` dicts, in object
        order (label 1 is meshes[0]), vertices in the unit of the pose translations."""
        from gigapose_b200.icp import device_meshes
        if not hasattr(self, "meshes"):
            self.meshes = {}
        self.meshes[dataset_name] = device_meshes(meshes, self.device if self.device.type == "cuda" else "cuda")

    @torch.no_grad()
    def refine_depth(self, dataset_name, predictions, depth, frame_idx=None, masks=None, hypotheses=1, *, K=None,
                     rank=False, mask_normals=False, refiner="icp", **params):
        """MegaPose's ICPRefiner.refine_poses on the output of `retrieve()`: the first `hypotheses` of the k poses of every
        detection are rendered and refined against the measured depth (gigapose_b200.icp.refine_icp).

        depth [F,H,W] (or [H,W]) measured depth in the unit of the poses, 0 = missing; frame_idx [B] frame of each
        detection (default: the `batch_im_id` column, or 0 for a single frame); masks None (threshold rule) or [B,H,W]
        full-frame detection masks; K, keyword only and required, the frames' full-image intrinsics [F,3,3] (or one
        [3,3] for all): `retrieve()`'s output does not carry them, and the batch's per-detection `tar_K` [B,3,3] is
        indexed by detection, not by frame (pass `tar_K[i]` of one detection i per frame); params as
        gigapose_b200.icp.DEFAULTS.  Returns a new collection: `pred_poses` replaced where the
        refinement was accepted (same order, nothing re-sorted), `poses_input` the coarse poses, and `icp_status`,
        `icp_residual`, `icp_fitness` [B,hypotheses].  With `rank=True` the final poses (refined where accepted, coarse
        where not) are also scored against the depth (gigapose_b200.icp.score_hypotheses, row f10) and the collection
        carries `depth_counts` [B,hypotheses,4] (consistent, behind, front, missing pixels), `depth_score`
        [B,hypotheses] and `best_hypothesis` [B] (int64: the highest score, the lowest index on a tie); the order of the
        hypotheses still does not change.

        With `mask_normals=True` (row f11, an extension: the reference smooths the whole frame) `masks` is required, one
        per detection, not per hypothesis: dense [B,H,W] or dict(counts=, offsets=) of COCO run-length masks
        (offsets [B+1], bop_run's layout); every hypothesis is refined against target normals smoothed within its
        detection's mask (gigapose_b200.icp.refine_icp_masked).

        With `refiner="teaserpp"` (row f13) the hypotheses go through MegaPose's TeaserppRefiner instead
        (gigapose_b200.teaser.refine_teaserpp, params as gigapose_b200.teaser.DEFAULTS) and the collection carries
        `teaser_status`, `teaser_inliers` and `teaser_clique` [B,hypotheses] in place of the ICP's three; `rank` works
        the same.  The reference's TEASER++ refiner takes no masks, so `masks` and `mask_normals` are refused with it."""
        from gigapose_b200.icp import refine_icp_masked, score_hypotheses
        from gigapose_b200.teaser import REFINERS
        if K is None:
            raise TypeError("refine_depth needs K=, the frames' full-image intrinsics [F,3,3] or [3,3]")
        if refiner not in REFINERS:
            raise ValueError(f"refiner must be {' or '.join(map(repr, REFINERS))}, got {refiner!r}")
        r = REFINERS[refiner]
        if not r.masks and (masks is not None or mask_normals):
            raise ValueError(f"refiner={refiner!r} takes no masks: the reference's refiner ignores them")
        meshes = self.meshes[dataset_name]
        poses = predictions.pred_poses
        B, k = poses.shape[:2]
        h = max(1, min(int(hypotheses), k))
        depth = torch.as_tensor(depth)
        n_frames = 1 if depth.dim() == 2 else depth.shape[0]
        if frame_idx is None:
            if "batch_im_id" in predictions.infos:
                frame_idx = np.asarray(predictions.infos.batch_im_id, np.int64)
            elif n_frames == 1:
                frame_idx = np.zeros(B, np.int64)
            else:
                raise ValueError("frame_idx is needed when depth holds several frames")
        frame_idx = np.asarray(torch.as_tensor(frame_idx).cpu()).reshape(-1)
        labels = np.repeat(object_indices(predictions.infos, len(meshes)), h)
        hyp_poses = poses[:, :h].reshape(-1, 4, 4)
        if mask_normals:
            if masks is None:
                raise ValueError("mask_normals=True needs masks, dense [B,H,W] or dict(counts=, offsets=)")
            dense, rle = (None, (masks["counts"], masks["offsets"])) if isinstance(masks, dict) else (masks, None)
            out, *extra = refine_icp_masked(meshes, labels, hyp_poses, depth, K, frame_idx, np.repeat(np.arange(B), h),
                                            dense, rle, **params)
        else:
            if masks is not None:
                params = dict(params, masks=torch.as_tensor(masks).to(poses.device).repeat_interleave(h, 0))
            out, *extra = r.refine(meshes, labels, hyp_poses, depth, K, np.repeat(frame_idx, h), **params)
        refined = predictions.clone()
        refined.register_tensor("poses_input", poses.clone())
        new = poses.clone()
        new[:, :h] = out.reshape(B, h, 4, 4)
        refined.register_tensor("pred_poses", new)
        for name, v in zip(r.outputs, extra):
            refined.register_tensor(name, v.reshape(B, h))
        if rank:
            counts, score, best = score_hypotheses(meshes, labels, out, depth, K, np.repeat(frame_idx, h), h,
                                                   unit_per_m=params.get("unit_per_m", r.defaults["unit_per_m"]))
            refined.register_tensor("depth_counts", counts.reshape(B, h, 4))
            refined.register_tensor("depth_score", score.reshape(B, h))
            refined.register_tensor("best_hypothesis", best.to(torch.int64))
        return refined

    # ------------------------------------------------------------------ localisation filter + writer (gigaPose.py:400-449)
    def filter_and_save(self, predictions, test_list, time, save_path, keep_only_testing_instances=True):
        labels = np.asarray(predictions.infos.label).astype(np.int32)
        assert len(np.unique(labels)) == len(np.unique(test_list.infos.obj_id))
        selected, detection_times = [], []
        if keep_only_testing_instances:
            top1 = predictions.scores[:, 0].detach().cpu().numpy()
            for row, obj_id in enumerate(test_list.infos.obj_id):
                n_inst = int(test_list.infos.inst_count[row])
                members = np.nonzero(labels == obj_id)[0]
                order = np.argsort(-top1[members], kind="stable")[:n_inst]
                selected.extend(members[order].tolist())
                detection_times.extend([test_list.infos.detection_time[row]] * n_inst)
        else:
            selected = list(range(len(labels)))
            detection_times = [0.0] * len(labels)
        predictions = predictions[selected]
        det_t = torch.as_tensor(np.asarray(detection_times), device=predictions.scores.device)
        predictions.register_tensor("detection_time", det_t)
        predictions.register_tensor("time", torch.ones_like(det_t) * time)
        np.savez(save_path,
                 scene_id=np.asarray(predictions.infos.scene_id).astype(np.int32),
                 im_id=np.asarray(predictions.infos.view_id).astype(np.int32),
                 object_id=np.asarray(predictions.infos.label).astype(np.int32),
                 time=predictions.time.cpu().numpy(), detection_time=predictions.detection_time.cpu().numpy(),
                 poses=predictions.pred_poses.cpu().numpy(), scores=predictions.scores.cpu().numpy())
        return selected, predictions

    # ------------------------------------------------------------------ the hot path (gigaPose.py:481-633)
    @torch.no_grad()
    def _retrieve_chunk(self, eng, tar_img, tar_mask, q_obj, tar_K, tar_M, mark=lambda name: None, sort=True):
        """Rows a1, a3-a9 for at most `eng.max_batch` detections; every step is a kernel launch on the current
        stream, no host synchronisation -> capturable as a CUDA graph."""
        mark("start")
        tokens = self.ae_net.raw_tokens(tar_img)                             # x_prenorm [b,257,1024]
        mark("a1_vit")
        eng.set_queries(tokens, tar_mask, q_obj, norm_passes=2)              # CLS drop, ae_net.py:69, matching.py:229 fused
        m = eng.sim_topk()
        mark("a3_a4_similarity_topk")
        tar_ist = self.ist_net.forward_by_chunk(tar_img)                     # once, not k times
        mark("a6_ist_backbone")
        rel_scale, rel_inplane = eng.ist_mlp(tar_ist, m)
        mark("a5_ist_mlp")
        r = eng.ransac(m, rel_scale, rel_inplane)
        out = eng.sort_and_pose(tar_K, tar_M, m, rel_scale, rel_inplane, r, sort_by_inliers=sort)
        mark("a7_a8_a9_ransac_sort_pose")
        return out

    GRAPH_BUCKET = 4          # batch sizes are padded to a multiple of this before graph capture / replay

    def _graphed_chunk(self, eng, dataset_name, tar_img, tar_mask, q_obj, tar_K, tar_M, sort=True):
        """Static input buffers + one captured graph per (dataset, padded batch size); outputs are copies of the graph's
        static tensors.  The reference's test loop hands over a different number of detections per image
        (test.py:55-60): batch sizes are padded to the next multiple of GRAPH_BUCKET by repeating the last detection
        (detections are independent, so the first B rows are unaffected) and the outputs sliced, which bounds the
        number of captures at max_dets_per_call / GRAPH_BUCKET."""
        B = tar_img.shape[0]
        Bp = min(-(-B // self.GRAPH_BUCKET) * self.GRAPH_BUCKET, eng.max_batch)
        key = (dataset_name, Bp, bool(sort))
        entry = self._graphs.get(key)
        args = (tar_img, tar_mask, q_obj, tar_K, tar_M)
        if entry is None:
            static = [torch.cat([t, t[-1:].expand(Bp - B, *t.shape[1:])]).contiguous() if Bp > B else t.clone() for t in args]
            side = torch.cuda.Stream(device=eng.device)
            side.wait_stream(torch.cuda.current_stream(eng.device))
            with torch.cuda.stream(side):
                for _ in range(2):                                           # warm-up outside the capture
                    self._retrieve_chunk(eng, *static, sort=sort)
            torch.cuda.current_stream(eng.device).wait_stream(side)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                out = self._retrieve_chunk(eng, *static, sort=sort)
            entry = (graph, static, out)
            self._graphs[key] = entry
        graph, static, out = entry
        for dst, src in zip(static, args):
            dst[:B].copy_(src, non_blocking=True)
            if Bp > B:
                dst[B:].copy_(src[-1:].expand(Bp - B, *src.shape[1:]), non_blocking=True)
        graph.replay()
        # the graph's static output tensors are overwritten by the next replay of the same batch size (the next chunk
        # of this call, or the next call): hand out copies (110 KB per detection)
        return {k: v[:B].clone() for k, v in out.items()}

    def stage(self, batch, dataset_name):
        """Start the host->device copy of a (pinned) batch on a dedicated copy stream and return the device-resident
        batch; `retrieve` waits for the copy.  Staging batch i+1 before retrieving batch i overlaps its upload with
        batch i's kernels (what a DataLoader with `pin_memory` + a prefetching trainer loop does for the reference)."""
        if dataset_name not in self.engines:
            self.set_template_data(dataset_name)
        device = self.engines[dataset_name].device
        if getattr(self, "_copy_stream", None) is None:
            self._copy_stream = torch.cuda.Stream(device=device)
        with torch.cuda.stream(self._copy_stream):
            staged = tc.PandasTensorCollection(infos=batch.infos, **{k: v.to(device, non_blocking=True)
                                                                     for k, v in batch._tensors.items()})
            # object indices (gigaPose.py:514-520) through a small ring of pinned buffers: a fresh `pin_memory()` per batch
            # goes through cudaHostAlloc, which was measured to stall the launching thread for up to 10 ms
            idx = object_indices(batch.infos, self.engines[dataset_name].O)
            ring = getattr(self, "_label_ring", None)
            if ring is None:
                ring = self._label_ring = {"slot": 0, "bufs": {}}
            ring["slot"] = (ring["slot"] + 1) % 4
            key = (ring["slot"], len(idx))
            labels = ring["bufs"].get(key)
            if labels is None:
                labels = ring["bufs"][key] = torch.empty(len(idx), dtype=torch.int64, pin_memory=True)
            labels.copy_(torch.from_numpy(idx))
            staged._q_obj = labels.to(device, non_blocking=True)
            ready = torch.cuda.Event()
            ready.record(self._copy_stream)
        staged._ready = ready
        for name in ("test_list",):
            if hasattr(batch, name):
                setattr(staged, name, getattr(batch, name))
        return staged

    def fetch_async(self, predictions):
        """Enqueue the device->host copy of a batch's poses and scores (pinned ring buffers, current stream) and return
        a handle whose `.result()` waits for it: the caller can launch the next batch before reading this one."""
        ring = getattr(self, "_host_ring", None)
        if ring is None:
            ring = self._host_ring = {"slot": 0, "bufs": {}}
        ring["slot"] = (ring["slot"] + 1) % 3
        out = []
        for name in ("pred_poses", "scores"):
            t = getattr(predictions, name)
            key = (name, ring["slot"], tuple(t.shape), t.dtype)
            buf = ring["bufs"].get(key)
            if buf is None:
                buf = ring["bufs"][key] = torch.empty(t.shape, dtype=t.dtype, pin_memory=True)
            buf.copy_(t, non_blocking=True)
            out.append(buf)
        done = torch.cuda.Event()
        done.record()
        return _HostResult(out[0], out[1], done)

    @torch.no_grad()
    def retrieve(self, batch, dataset_name, sort_pred_by_inliers=True):
        """Rows a1, a3-a9 for one batch; returns the PandasTensorCollection `eval_retrieval` builds."""
        if dataset_name not in self.engines:
            self.set_template_data(dataset_name)
        eng = self.engines[dataset_name]
        device = eng.device
        ready = getattr(batch, "_ready", None)
        if ready is not None:                            # staged batch: its upload ran on the copy stream
            cur = torch.cuda.current_stream(device)
            cur.wait_event(ready)
            for t in list(batch._tensors.values()) + [batch._q_obj]:
                t.record_stream(cur)
        tar_img = batch.tar_img.to(device, non_blocking=True)
        tar_mask = batch.tar_mask.to(device, non_blocking=True)
        if ready is not None:
            q_obj = batch._q_obj                         # uploaded with the batch: no blocking pageable copy here
        else:
            q_obj = torch.as_tensor(object_indices(batch.infos, eng.O), device=device)   # gigaPose.py:514-520
        tar_K, tar_M = batch.tar_K.to(device).float(), batch.tar_M.to(device).float()
        outs = []
        B = tar_img.shape[0]
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        marks = []

        def mark(name):
            if self.profile_stages:
                e = torch.cuda.Event(enable_timing=True)
                e.record()
                marks.append((name, e))

        for b0 in range(0, B, eng.max_batch):
            sl = slice(b0, min(B, b0 + eng.max_batch))
            args = (tar_img[sl], tar_mask[sl], q_obj[sl], tar_K[sl], tar_M[sl])
            if self.use_cuda_graph and not self.profile_stages:
                outs.append(self._graphed_chunk(eng, dataset_name, *args, sort=sort_pred_by_inliers))
            else:
                outs.append(self._retrieve_chunk(eng, *args, mark=mark, sort=sort_pred_by_inliers))
        ev[1].record()
        if self.profile_stages:
            torch.cuda.synchronize(device)
            self.stage_ms = {}
            for (n0, e0), (n1, e1) in zip(marks[:-1], marks[1:]):
                if n1 != "start":
                    self.stage_ms[n1] = self.stage_ms.get(n1, 0.0) + e0.elapsed_time(e1)
        out = outs[0] if len(outs) == 1 else {k: torch.cat([o[k] for o in outs], 0) for k in outs[0]}
        self._events = ev
        return tc.PandasTensorCollection(infos=batch.infos, **out)

    def eval_retrieval(self, batch, idx_batch, dataset_name, sort_pred_by_inliers=True):
        predictions = self.retrieve(batch, dataset_name, sort_pred_by_inliers=sort_pred_by_inliers)
        ev = self._events
        ev[1].synchronize()
        # CUDA-event time of the whole retrieval.  (The reference's wall-clock timer is overwritten between its two
        # `tic()`s and never counts the ViT + similarity stages, SURVEY §5; here the saved `time` covers everything.)
        total_time = ev[0].elapsed_time(ev[1]) / 1e3
        self.last_times = {"retrieval": total_time}
        save_path = osp.join(self.log_dir, "predictions", f"{idx_batch}.npz")
        test_list = getattr(batch, "test_list", None)
        if test_list is None:                      # synthetic / detection-style batches: nothing to filter against
            return list(range(len(predictions))), predictions
        return self.filter_and_save(predictions, test_list=test_list, time=total_time, save_path=save_path)

    @torch.no_grad()
    def test_step(self, batch, idx_batch):
        self.eval_retrieval(batch, idx_batch=idx_batch, dataset_name=self.test_dataset_name)
        return 0

    def on_test_epoch_end(self):
        if self.global_rank != 0:
            return
        prediction_dir = osp.join(self.log_dir, "predictions")
        from src.utils.inout import save_predictions_from_batched_predictions      # row f4: BOP csv export
        save_predictions_from_batched_predictions(prediction_dir, dataset_name=self.test_dataset_name,
                                                  model_name=self.model_name, run_id=self.run_id, is_refined=False)
