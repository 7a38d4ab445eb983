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
        return self._onboard(dataset_name, len(rgba), rgba[0].shape[0],
                             lambda o: (rgba[o].to(self.device, non_blocking=True).float(), boxes[o]), K, poses)

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

        def produce(o):
            mesh = read_ply(meshes[o]) if isinstance(meshes[o], (str, os.PathLike)) else meshes[o]
            r = render_templates(mesh, poses[o].to(self.device), K, device=self.device)
            return r["rgba"], r["boxes"]

        return self._onboard(dataset_name, n_obj, poses.shape[1], produce, K, poses)

    def _onboard(self, dataset_name, n_obj, T, produce, K, poses):
        """The body of both onboarding entry points: `produce(o)` -> (rgba [T,4,H,W] f32 on the device, boxes [T,4])."""
        from gigapose_b200.engine import Engine
        from gigapose_b200.preprocess import CLIP_MEAN, CLIP_STD, crop_resize_pad
        device = self.device
        metric = self.testing_metric
        eng = Engine(n_obj, T, self.max_dets_per_call, device=device, k=metric.k, sim_threshold=metric.sim_threshold,
                     patch_threshold=metric.patch_threshold, precision=getattr(metric, "precision", "fp32_split"))
        start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        builder = _BankBuilder(self, eng)
        Ms = []
        for o in range(n_obj):
            rgba, boxes = produce(o)
            crop = crop_resize_pad(torch.as_tensor(boxes), rgba, 224,
                                   mean=CLIP_MEAN + (0.0,), std=CLIP_STD + (1.0,))      # alpha channel passes through
            builder.add(o, crop["images"][:, :3], crop["images"][:, 3])
            Ms.append(crop["M"])
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
        self.onboarding_s_per_object = start.elapsed_time(stop) / 1e3 / n_obj
        logger.info(f"Onboarded {dataset_name}: {n_obj} objects x {T} templates, {self.onboarding_s_per_object:.3f} s/object")
        return eng

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
