"""Host-side handle over the C ABI: owns the template bank + workspace as torch-allocated HBM and launches the
sm_90a kernels on torch's current stream.  PyTorch is used for device memory, streams and torch.distributed only;
every arithmetic step below is a kernel of libgigapose_b200.so (no torch fallback)."""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import torch

from . import _lib
from ._lib import (GpCandidates, GpConfig, GpMatches, GpPredictions, GpRansacOut, LAYOUT_CHANNEL_MAJOR,
                   LAYOUT_PATCH_MAJOR, LAYOUT_VIT_TOKENS, PRECISION_BF16, PRECISION_FP32_SPLIT, check, ptr)

P = 256
C_AE = 1024
C_IST = 256


def _f32(t: torch.Tensor, device) -> torch.Tensor:
    if t.device != device:
        t = t.to(device, non_blocking=True)
    if t.dtype != torch.float32:
        t = t.float()
    return t


def _feature_layout(feat: torch.Tensor):
    """Accepts [n,C,16,16] (reference layout) or [n,256,C] (patch-major).  A channels-last *view* of a patch-major
    buffer (what AENet returns) is recognised and used in place, without a copy."""
    if feat.dim() == 4:
        n, c, h, w = feat.shape
        assert h * w == P, f"expected a 16x16 patch grid, got {h}x{w}"
        if feat.stride() == (P * c, 1, w * c, c):          # [n,16,16,C] memory viewed as [n,C,16,16]
            return feat, LAYOUT_PATCH_MAJOR
        return feat.contiguous(), LAYOUT_CHANNEL_MAJOR
    if feat.dim() == 3 and feat.shape[1] == P + 1:         # raw ViT tokens [n,257,C] (`x_prenorm`): CLS row skipped in-kernel
        return feat.contiguous(), LAYOUT_VIT_TOKENS
    assert feat.dim() == 3 and feat.shape[1] == P, f"bad descriptor shape {tuple(feat.shape)}"
    return feat.contiguous(), LAYOUT_PATCH_MAJOR


def _ist_layout(feat: torch.Tensor):
    """[n,256,16,16] IST features; the channels-last view the native trunk returns ([n,16,16,256] memory) is taken in
    place as patch-major, anything else is made contiguous channel-major."""
    n, c, h, w = feat.shape
    assert (c, h * w) == (C_IST, P), tuple(feat.shape)
    if feat.stride() == (P * c, 1, w * c, c):
        return feat, LAYOUT_PATCH_MAJOR
    return feat.contiguous(), LAYOUT_CHANNEL_MAJOR


def ransac_points(lib, src_pts, tar_pts, rel_scale, rel_inplane, out, pixel_threshold, patch_size, stream):
    """gp_ransac over n = prod(leading dims) (detection, hypothesis) pairs; tensors [..., 256, 2] / [..., 256]."""
    n = src_pts.numel() // (P * 2)
    rs = Engine._ransac_struct(out)
    check(lib.gp_ransac(n, float(pixel_threshold), int(patch_size), src_pts.data_ptr(), tar_pts.data_ptr(),
                        rel_scale.data_ptr(), rel_inplane.data_ptr(), C.byref(rs), stream))


class Engine:
    """One template bank (or one shard of it) resident on one GPU plus the per-batch workspace."""

    def __init__(self, num_objects: int, num_templates: int, max_batch: int, device="cuda:0", k: int = 5,
                 sim_threshold: float = 0.5, patch_threshold: float = 3, pixel_threshold: float = 14.0,
                 patch_size: int = 14, precision: str = "fp32_split", shard_rank: int = 0, shard_world: int = 1,
                 num_templates_global: Optional[int] = None, ist_bank_global: bool = False):
        self.lib = _lib.load()
        self.device = _lib.cuda_device(device, "gigapose_b200 runs")
        self.k = int(k)
        self.O, self.T, self.max_batch = int(num_objects), int(num_templates), int(max_batch)
        self.T_global = int(num_templates_global if num_templates_global is not None else num_templates)
        self.shard_rank, self.shard_world = int(shard_rank), int(shard_world)
        cfg = GpConfig(abi_version=_lib.GP_ABI_VERSION, device=self.device.index, num_objects=self.O,
                       num_templates=self.T, num_templates_global=self.T_global,
                       template_id_stride=self.shard_world, template_id_offset=self.shard_rank,
                       max_batch=self.max_batch, top_k=self.k, sim_threshold=float(sim_threshold),
                       patch_threshold=float(patch_threshold), pixel_threshold=float(pixel_threshold),
                       patch_size=int(patch_size),
                       precision={"fp32_split": PRECISION_FP32_SPLIT, "bf16": PRECISION_BF16}[precision],
                       ist_bank_global=1 if ist_bank_global else 0)
        self.ist_bank_global = bool(ist_bank_global)
        self.cfg = cfg
        self.precision = precision
        bank_b, ws_b = C.c_size_t(), C.c_size_t()
        check(self.lib.gp_query_sizes(C.byref(cfg), C.byref(bank_b), C.byref(ws_b)))
        self.bank_bytes, self.workspace_bytes = bank_b.value, ws_b.value
        self._bank_mem, self._bank = _lib.aligned_buffer(self.bank_bytes, self.device, zero=True)
        self._ws_mem, ws = _lib.aligned_buffer(self.workspace_bytes, self.device)
        h = C.c_void_p()
        check(self.lib.gp_create(C.byref(cfg), self._bank.data_ptr(), ws.data_ptr(), C.byref(h)))
        self._h = h
        self._keep = []          # tensors whose device pointers the library retains
        self._B = 0

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            try:
                self.lib.gp_destroy(h)
            except Exception:
                pass
            self._h = None

    # ------------------------------------------------------------------------------------------------ helpers
    @property
    def stream(self) -> int:
        return torch.cuda.current_stream(self.device).cuda_stream

    def _empty(self, shape, dtype):
        return torch.empty(shape, dtype=dtype, device=self.device)

    # ---------------------------------------------------------------------------------------------- onboarding
    def bank_write(self, obj: int, tmpl0: int, feat: torch.Tensor, mask: torch.Tensor,
                   ist_feat: Optional[torch.Tensor] = None, norm_passes: int = 1) -> None:
        """feat: [n,1024,16,16], [n,256,1024] or raw ViT tokens [n,257,1024] (use norm_passes=2); mask: [n,H,W];
        ist_feat: [n,256,16,16] (optional)."""
        feat, layout = _feature_layout(_f32(feat, self.device))
        mask = _f32(mask, self.device).contiguous()
        n = feat.shape[0]
        assert mask.shape[0] == n and mask.dim() == 3
        check(self.lib.gp_bank_write(self._h, obj, tmpl0, n, feat.data_ptr(), layout, norm_passes, mask.data_ptr(),
                                     mask.shape[1], mask.shape[2], None, self.stream))
        if ist_feat is not None:
            assert ist_feat.shape[0] == n
            if self.ist_bank_global:
                raise _lib.GigaPoseNativeError("ist_bank_global engine: write IST features with bank_write_ist(global ids)")
            self.bank_write_ist(obj, tmpl0, ist_feat)

    def bank_write_ist(self, obj: int, tmpl0: int, ist_feat: torch.Tensor) -> None:
        """IST features [n,256,16,16] into IST-bank slots [tmpl0, tmpl0+n) of object `obj` (GLOBAL template ids when
        the engine was created with `ist_bank_global=True`)."""
        ist_feat, layout = _ist_layout(_f32(ist_feat, self.device))
        check(self.lib.gp_bank_write_ist(self._h, obj, tmpl0, ist_feat.shape[0], ist_feat.data_ptr(), layout, self.stream))

    def set_poses(self, K: torch.Tensor, M: torch.Tensor, poses: torch.Tensor) -> None:
        K, M, poses = (_f32(x, self.device).contiguous() for x in (K, M, poses))
        assert K.shape == (self.O, 3, 3) and M.shape == (self.O, self.T_global, 3, 3)
        assert poses.shape == (self.O, self.T_global, 4, 4)
        check(self.lib.gp_bank_set_poses(self._h, K.data_ptr(), M.data_ptr(), poses.data_ptr(), self.stream))

    # ---------------------------------------------------------------------------------------- persistence (row f2)
    BANK_MAGIC = b"GPB200BANK\x00"
    BANK_FORMAT = 1

    def _bank_view(self) -> torch.Tensor:
        """The bank as the library carves it: `bank_bytes` bytes from the 1024-aligned base."""
        return self._bank

    def _bank_header(self) -> dict:
        c = self.cfg
        return dict(format=self.BANK_FORMAT, abi_version=int(c.abi_version), num_objects=self.O, num_templates=self.T,
                    num_templates_global=self.T_global, template_id_stride=self.shard_world,
                    template_id_offset=self.shard_rank, precision=self.precision, patch_size=int(c.patch_size),
                    ist_bank_global=int(self.ist_bank_global), bank_bytes=int(self.bank_bytes),
                    fingerprint=getattr(self, "fingerprint", ""))

    def save_bank(self, path: str) -> None:
        """Writes the onboarded bank -- descriptor planes, sampled masks, IST features and pose tables exactly as they
        lie in HBM (the library carves one caller-owned buffer at fixed offsets, so the bytes are position independent)
        -- behind a small JSON header.  The reference only caches raw template crops
        (custom_megapose/template_dataset.py:91-119) and re-encodes them at every start (gigaPose.py:357-398)."""
        import json
        header = json.dumps(self._bank_header(), sort_keys=True).encode()
        host = self._bank_view().cpu().numpy()                    # stream-ordered copy + sync
        tmp = path + ".tmp"
        with open(tmp, "wb") as f:
            f.write(self.BANK_MAGIC)
            f.write(len(header).to_bytes(8, "little"))
            f.write(header)
            host.tofile(f)
        os.replace(tmp, path)

    def load_bank(self, path: str) -> None:
        """Inverse of `save_bank`; refuses files written for another shape / shard / precision / library ABI."""
        import json
        import numpy as np
        with open(path, "rb") as f:
            if f.read(len(self.BANK_MAGIC)) != self.BANK_MAGIC:
                raise _lib.GigaPoseNativeError(f"{path} is not a gigapose_b200 bank file")
            header = json.loads(f.read(int.from_bytes(f.read(8), "little")))
            want = self._bank_header()
            if header != want:
                diff = {k: (header.get(k), v) for k, v in want.items() if header.get(k) != v}
                raise _lib.GigaPoseNativeError(f"bank file {path} does not match this engine: {diff}")
            data = np.fromfile(f, dtype=np.uint8)
        if data.size != self.bank_bytes:
            raise _lib.GigaPoseNativeError(f"bank file {path} is truncated: {data.size} of {self.bank_bytes} bytes")
        self._bank_view().copy_(torch.from_numpy(data))

    def set_ist_weights(self, regressor) -> None:
        """`regressor`: module with `scale_predictor` / `inplane_predictor` Sequentials (ist_net.py:140-155)."""
        ws = []
        for head in (regressor.scale_predictor, regressor.inplane_predictor):
            for idx in (0, 2, 4):
                # engine-owned copies (3 MB): the library retains raw pointers, which must not alias module parameters
                # that a later `.to()` / `.half()` / load_state_dict could free or rewrite
                ws.append(_f32(head[idx].weight.detach(), self.device).clone(memory_format=torch.contiguous_format))
                ws.append(_f32(head[idx].bias.detach(), self.device).clone(memory_format=torch.contiguous_format))
        assert ws[0].shape == (512, 512) and ws[2].shape == (256, 512) and ws[4].shape == (1, 256)
        assert ws[6].shape == (512, 512) and ws[8].shape == (256, 512) and ws[10].shape == (2, 256)
        self._keep = ws
        arr = (C.c_void_p * 12)(*[w.data_ptr() for w in ws])
        use_tanh = 1 if isinstance(regressor.inplane_predictor[-1], torch.nn.Tanh) else 0
        check(self.lib.gp_set_ist_weights(self._h, arr, use_tanh, self.stream))

    # ------------------------------------------------------------------------------------------------ per batch
    def set_queries(self, q_feat: torch.Tensor, q_mask: torch.Tensor, q_obj: torch.Tensor, norm_passes: int = 1) -> None:
        q_feat, layout = _feature_layout(_f32(q_feat, self.device))
        q_mask = _f32(q_mask, self.device).contiguous()
        q_obj = q_obj.to(self.device, dtype=torch.int32).contiguous()
        B = q_feat.shape[0]
        assert q_mask.shape[0] == B and q_obj.shape == (B,)
        check(self.lib.gp_set_queries(self._h, B, q_feat.data_ptr(), layout, norm_passes, q_mask.data_ptr(),
                                      q_mask.shape[1], q_mask.shape[2], q_obj.data_ptr(), self.stream))
        self._B = B

    def _alloc_matches(self, B):
        k = self.k
        return dict(id_src=self._empty((B, k), torch.int64), score_src=self._empty((B, k), torch.float32),
                    score_pts=self._empty((B, k, P), torch.float32), tar_pts=self._empty((B, k, P, 2), torch.int64),
                    src_pts=self._empty((B, k, P, 2), torch.int64))

    @staticmethod
    def _matches_struct(m) -> GpMatches:
        return GpMatches(m["id_src"].data_ptr(), m["score_src"].data_ptr(), m["score_pts"].data_ptr(),
                         m["tar_pts"].data_ptr(), m["src_pts"].data_ptr())

    def alloc_candidates(self, B, G=1):
        k = self.k
        return dict(score=self._empty((G, B, k), torch.float32), id=self._empty((G, B, k), torch.int32),
                    pts_score=self._empty((G, B, k, P), torch.float32), idx=self._empty((G, B, k, P), torch.uint8),
                    valid=self._empty((G, B, k, P), torch.uint8))

    @staticmethod
    def _cand_struct(c) -> GpCandidates:
        return GpCandidates(c["score"].data_ptr(), c["id"].data_ptr(), c["pts_score"].data_ptr(), c["idx"].data_ptr(),
                            c["valid"].data_ptr(), ptr(c.get("rel_scale")), ptr(c.get("rel_inplane")))

    def sim_topk(self) -> Dict[str, torch.Tensor]:
        """LocalSimilarity.test on the staged queries against the resident bank (single GPU)."""
        m = self._alloc_matches(self._B)
        ms = self._matches_struct(m)
        check(self.lib.gp_sim_topk(self._h, self._B, C.byref(ms), self.stream))
        return m

    def sim_candidates(self, out=None) -> Dict[str, torch.Tensor]:
        c = out if out is not None else self.alloc_candidates(self._B)
        cs = self._cand_struct(c)
        check(self.lib.gp_sim_candidates(self._h, self._B, C.byref(cs), self.stream))
        return c

    def topk_merge(self, gathered: Dict[str, torch.Tensor], G: int, rank_stride_bytes: int = 0):
        """Global top-k over G candidate lists.  Returns the matches and, when the candidates carry the per-shard IST
        outputs, the winners' (rel_scale, rel_inplane)."""
        B = self._B
        m = self._alloc_matches(B)
        cs, ms = self._cand_struct(gathered), self._matches_struct(m)
        rs = ri = None
        if gathered.get("rel_scale") is not None:
            rs = self._empty((B, self.k, P), torch.float32)
            ri = self._empty((B, self.k, P, 2), torch.float32)
        check(self.lib.gp_topk_merge(self._h, B, G, C.byref(cs), rank_stride_bytes, C.byref(ms), ptr(rs), ptr(ri),
                                     self.stream))
        return (m, rs, ri) if rs is not None else m

    def ist_mlp(self, q_ist: torch.Tensor, matches: Dict[str, torch.Tensor], b0: int = 0):
        """Row a5 for the detections [b0, b0+n) of the staged batch; `q_ist` [n,256,16,16] and `matches` are
        window-relative (n = their leading dimension)."""
        q_ist, layout = _ist_layout(_f32(q_ist, self.device))
        n = q_ist.shape[0]
        assert matches["id_src"].shape[0] == n
        rel_scale = self._empty((n, self.k, P), torch.float32)
        rel_inplane = self._empty((n, self.k, P, 2), torch.float32)
        ms = self._matches_struct(matches)
        check(self.lib.gp_ist_mlp(self._h, b0, n, q_ist.data_ptr(), layout, C.byref(ms), rel_scale.data_ptr(),
                                  rel_inplane.data_ptr(), self.stream))
        return rel_scale, rel_inplane

    def _alloc_ransac(self, B):
        k = self.k
        return dict(M=self._empty((B, k, 3, 3), torch.float32), idx_failed=self._empty((B, k), torch.uint8),
                    ransac_src_pts=self._empty((B, k, P, 2), torch.int64),
                    ransac_tar_pts=self._empty((B, k, P, 2), torch.int64),
                    ransac_scores=self._empty((B, k, P), torch.int64), inlier_count=self._empty((B, k), torch.int32))

    @staticmethod
    def _ransac_struct(r) -> GpRansacOut:
        return GpRansacOut(r["M"].data_ptr(), r["idx_failed"].data_ptr(), r["ransac_src_pts"].data_ptr(),
                           r["ransac_tar_pts"].data_ptr(), r["ransac_scores"].data_ptr(),
                           r["inlier_count"].data_ptr() if "inlier_count" in r else None)

    def ransac(self, matches, rel_scale, rel_inplane) -> Dict[str, torch.Tensor]:
        B = matches["src_pts"].shape[0]
        r = self._alloc_ransac(B)
        ransac_points(self.lib, matches["src_pts"], matches["tar_pts"], rel_scale, rel_inplane, r,
                      self.cfg.pixel_threshold, self.cfg.patch_size, self.stream)
        return r

    def sort_and_pose(self, q_K, q_M, matches, rel_scale, rel_inplane, ransac, b0: int = 0,
                      sort_by_inliers: bool = True) -> Dict[str, torch.Tensor]:
        """Rows a8 + a9 for the detections [b0, b0+n) of the staged batch (all tensors window-relative)."""
        k = self.k
        B = matches["id_src"].shape[0]
        q_K, q_M = _f32(q_K, self.device).contiguous(), _f32(q_M, self.device).contiguous()
        assert q_K.shape[0] == B and q_M.shape[0] == B
        out = self._alloc_matches(B)
        out.update(relScale=self._empty((B, k, P), torch.float32), relInplane=self._empty((B, k, P, 2), torch.float32))
        ro = self._alloc_ransac(B)
        ro.pop("inlier_count")
        out.update(ro)
        out.update(scores=self._empty((B, k), torch.float32), pred_poses=self._empty((B, k, 4, 4), torch.float32))
        pred = GpPredictions(self._matches_struct(out), out["relScale"].data_ptr(), out["relInplane"].data_ptr(),
                             self._ransac_struct(out), out["scores"].data_ptr(), out["pred_poses"].data_ptr())
        ms, rs = self._matches_struct(matches), self._ransac_struct(ransac)
        check(self.lib.gp_sort_and_pose(self._h, b0, B, 1 if sort_by_inliers else 0, q_K.data_ptr(), q_M.data_ptr(),
                                        C.byref(ms), rel_scale.data_ptr(), rel_inplane.data_ptr(), C.byref(rs),
                                        C.byref(pred), self.stream))
        out["idx_failed"] = out["idx_failed"].bool()
        return out

    # ------------------------------------------------------------------------------------------------ multi-GPU
    def comm_init(self, nccl_comm_ptr: int) -> None:
        """Binds an ncclComm_t (integer address, e.g. `ProcessGroupNCCL._comm_ptr()`) whose rank / size equal this
        engine's shard map."""
        check(self.lib.gp_comm_init(self._h, C.c_void_p(nccl_comm_ptr), self.shard_rank, self.shard_world))

    def allgather(self, send: torch.Tensor, recv: torch.Tensor) -> torch.Tensor:
        assert send.is_contiguous() and recv.is_contiguous()
        nbytes = send.numel() * send.element_size()
        assert recv.numel() * recv.element_size() == nbytes * self.shard_world
        check(self.lib.gp_allgather(self._h, send.data_ptr(), recv.data_ptr(), nbytes, self.stream))
        return recv

    def topk_allgather_merge(self, packed: torch.Tensor, rank_stride_bytes: int, slot0: Dict[str, torch.Tensor]):
        """In-place all-gather of the packed candidate records + global top-k merge (the collective of the search)."""
        B = self._B
        m = self._alloc_matches(B)
        cs, ms = self._cand_struct(dict(slot0, rel_scale=None, rel_inplane=None)), self._matches_struct(m)
        check(self.lib.gp_topk_allgather_merge(self._h, B, packed.data_ptr(), rank_stride_bytes, C.byref(cs),
                                               C.byref(ms), self.stream))
        return m

    def retrieve(self, q_feat, q_mask, q_obj, q_ist, q_K, q_M, norm_passes: int = 1) -> Dict[str, torch.Tensor]:
        """Rows a3-a9 for one batch on one GPU: the tensor content of GigaPose.eval_retrieval (gigaPose.py:497-604)."""
        self.set_queries(q_feat, q_mask, q_obj, norm_passes=norm_passes)
        m = self.sim_topk()
        rel_scale, rel_inplane = self.ist_mlp(q_ist, m)
        r = self.ransac(m, rel_scale, rel_inplane)
        return self.sort_and_pose(q_K, q_M, m, rel_scale, rel_inplane, r)

    # ---------------------------------------------------------------------------------------------- diagnostics
    def time_sim_kernel(self, iters: int = 10) -> float:
        ms = C.c_float()
        check(self.lib.gp_time_sim_kernel(self._h, self._B, iters, C.byref(ms), self.stream))
        return ms.value

    def debug_sim_tiles(self) -> torch.Tensor:
        """Raw fp32 similarity tiles [T, B(sorted by object), 256 t, 256 s] (tests only: 256 KiB per tile)."""
        tiles = self._empty((self.T, self._B, P, P), torch.float32)
        check(self.lib.gp_debug_sim_tiles(self._h, self._B, tiles.data_ptr(), self.stream))
        return tiles

    def launch_count(self) -> int:
        return int(self.lib.gp_launch_count())

    # algorithmic work of one similarity launch (SURVEY.md §8d): 2*T*P^2*C per detection
    def sim_flops(self, B: Optional[int] = None) -> float:
        return 2.0 * (B or self._B) * self.T * P * P * C_AE


# ------------------------------------------------------------------------------------------------------------
# explicit-input entry points behind the reference's module-level APIs (no resident bank): a cached scratch
# Engine with one "object" per query holds the gathered templates, exactly like the reference's per-call gather
# ------------------------------------------------------------------------------------------------------------
_SCRATCH = {}


def _scratch_engine(device, B, T, k, **cfg) -> Engine:
    key = (str(device), B, T, k, tuple(sorted(cfg.items())))
    eng = _SCRATCH.get(key)
    if eng is None:
        _SCRATCH.clear()                      # keep at most one scratch bank alive
        eng = Engine(B, T, B, device=device, k=k, **cfg)
        _SCRATCH[key] = eng
    return eng


def similarity_search_explicit(src_feats, tar_feat, src_masks, tar_mask, k, sim_threshold, patch_threshold,
                               precision="fp32_split") -> Dict[str, torch.Tensor]:
    """LocalSimilarity.test on explicit tensors: src_feats [B,N,C,16,16], tar_feat [B,C,16,16],
    src_masks [B,N,H,W], tar_mask [B,H,W] (matching.py:188-316)."""
    B, N = src_feats.shape[:2]
    eng = _scratch_engine(src_feats.device, B, N, k, sim_threshold=sim_threshold, patch_threshold=patch_threshold,
                          precision=precision)
    for b in range(B):
        eng.bank_write(b, 0, src_feats[b], src_masks[b], norm_passes=1)
    eng.set_queries(tar_feat, tar_mask, torch.arange(B, device=src_feats.device), norm_passes=1)
    return eng.sim_topk()


def ist_mlp_explicit(regressor, src_feat, tar_feat, src_pts, tar_pts):
    """ISTNet.inference on explicit tensors (ist_net.py:97-120): src_feat/tar_feat [B,256,16,16], pts [B,N,2]."""
    B, N = src_pts.shape[:2]
    assert N == P, "one correspondence slot per patch"
    dev = src_feat.device
    eng = _scratch_engine(dev, B, 1, 1)
    eng.set_ist_weights(regressor)
    ist = _f32(src_feat, eng.device).contiguous()
    zeros_feat = torch.zeros(1, P, C_AE, device=eng.device)
    ones_mask = torch.ones(1, 16, 16, device=eng.device)
    for b in range(B):
        eng.bank_write(b, 0, zeros_feat, ones_mask, ist_feat=ist[b:b + 1], norm_passes=0)
    eng.set_queries(torch.zeros(B, P, C_AE, device=eng.device), torch.ones(B, 16, 16, device=eng.device),
                    torch.arange(B, device=eng.device), norm_passes=0)
    m = dict(id_src=torch.zeros(B, 1, dtype=torch.int64, device=eng.device),
             src_pts=src_pts.to(eng.device).reshape(B, 1, P, 2).contiguous(),
             tar_pts=tar_pts.to(eng.device).reshape(B, 1, P, 2).contiguous(),
             score_src=torch.zeros(B, 1, device=eng.device), score_pts=torch.zeros(B, 1, P, device=eng.device))
    rs, ri = eng.ist_mlp(tar_feat, m)
    return rs.reshape(B, P), ri.reshape(B, P, 2)
