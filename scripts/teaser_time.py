"""Stage times of the TEASER++ depth refiner (row f13) beside the ICP (row f6) on the same hypotheses, on the cases of
scripts/icp_time.py (c2-shaped: 32 detections of 8 objects in 4 frames at 640 x 480) and scripts/bop_refine_time.py
(one LM-O-shaped 640 x 480 image of 8 instances and one HOPE-shaped 1920 x 1080 image of 18), for 1 and 5 hypotheses per
detection, the coarse poses perturbed as those scripts plant them (2-6 degrees, up to 8 mm per axis).  Stages, from CUDA
events, the median of 5 repetitions after a warm-up:
  render      `icp.render_hypotheses` of the coarse poses (shared by both refiners)
  compaction  gp_teaser_refine stopped after the points (debug.stop_after = 1)
  fps, graph, clique, solve   the differences of the runs stopped after sampling (2), the graph and order (3), the
              clique (4), and the full run (0): solve = GNC-TLS, voting and the inlier count
  teaser      the full gp_teaser_refine
  icp         gp_icp_prepare_scene + gp_icp_refine on the same renders
with the TEASER++ status counts (budget hits included), the mean clique size and clique-search nodes, the mean
translation / rotation error of the accepted poses and of the ICP's, and the card's name, power limit and clocks.

    python scripts/teaser_time.py [--out results/teaser_time.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from gigapose_b200 import bop_eval, icp, teaser  # noqa: E402
from icp_time import make_case, perturbed  # noqa: E402
from bop_refine_time import SHAPES, make_image  # noqa: E402

DEV = "cuda:0"
REPS = 5
STATUS = ["ok", "too_few_points", "clique_too_small", "clique_budget", "too_few_inliers", "invalid"]


def errors(P, truth):
    dt = np.linalg.norm(P[:, :3, 3] - truth[:, :3, 3], axis=1)
    dR = np.einsum("nji,njk->nik", P[:, :3, :3].astype(np.float64), truth[:, :3, :3].astype(np.float64))
    return dt, np.degrees(np.arccos(np.clip((np.trace(dR, axis1=1, axis2=2) - 1) / 2, -1, 1)))


def time_case(dm, labels, frames, T0, truth, depth, K):
    F, H, W = depth.shape
    n = len(T0)
    T0 = torch.as_tensor(T0).to(DEV)
    lab, fr = torch.as_tensor(labels), torch.as_tensor(frames)
    fi = fr.to(DEV, torch.int32)
    ws = torch.empty(icp.workspace_bytes(F, n, H, W), dtype=torch.uint8, device=DEV)
    counts = torch.zeros(n, 4, dtype=torch.int32, device=DEV)
    ms = {k: [] for k in ("render", "stop1", "stop2", "stop3", "stop4", "teaser", "icp")}
    for rep in range(REPS + 1):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(8)]
        ev[0].record()
        R, boxes = icp.render_hypotheses(dm, lab, T0, K, fr, H, W)
        ev[1].record()
        for s in (1, 2, 3, 4):
            teaser.refine_rendered(depth, K, fi, R, boxes, T0, debug=dict(stop_after=s))
            ev[1 + s].record()
        out = teaser.refine_rendered(depth, K, fi, R, boxes, T0, debug=dict(counts=counts))
        ev[6].record()
        icp.prepare_scene(depth, K, ws)
        iout = icp.refine_rendered(depth, K, fi, R, boxes, T0, None, ws)
        ev[7].record()
        torch.cuda.synchronize()
        if rep:
            for k, (a, b) in zip(ms, zip(ev[:-1], ev[1:])):
                ms[k].append(a.elapsed_time(b))
    med = {k: float(np.median(v)) for k, v in ms.items()}
    stages = dict(render=med["render"], compaction=med["stop1"], fps=med["stop2"] - med["stop1"],
                  graph=med["stop3"] - med["stop2"], clique=med["stop4"] - med["stop3"],
                  solve=med["teaser"] - med["stop4"], teaser=med["teaser"], icp=med["icp"])
    st = out[1].cpu().numpy()
    c = counts.cpu().numpy()
    ok = st == 0
    P, Pi = out[0].cpu().numpy(), iout[0].cpu().numpy()
    truth = np.repeat(truth, n // len(truth), 0)
    e0, et, ei = errors(T0.cpu().numpy(), truth), errors(P, truth), errors(Pi, truth)
    iok = iout[1].cpu().numpy() == 0
    return dict(ms=stages, status_counts=dict(zip(STATUS, np.bincount(st, minlength=6).tolist())),
                mean_clique=float(out[3].float().mean()), mean_nodes=float(c[:, 2].mean()), max_nodes=int(c[:, 2].max()),
                mean_gnc_iterations=float(c[ok, 3].mean()) if ok.any() else None,
                coarse_error=[float(e0[0].mean()), float(e0[1].mean())],
                teaser_accepted_error=[float(et[0][ok].mean()), float(et[1][ok].mean())] if ok.any() else None,
                icp_ok=int(iok.sum()), icp_accepted_error=[float(ei[0][iok].mean()), float(ei[1][iok].mean())]
                if iok.any() else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "teaser_time.py measures on a GPU"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    result = dict(device=torch.cuda.get_device_name(0), nvidia_smi=smi[0] if smi else None, cases={})
    rng = np.random.default_rng(1)
    dm, labels, frames, truth, depth, K = make_case(torch.device(DEV))
    for hyp in (1, 5):
        r = time_case(dm, np.repeat(labels, hyp), np.repeat(frames, hyp), perturbed(truth, hyp, rng), truth, depth, K)
        r["ms_per_detection"] = {k: v / len(truth) for k, v in r["ms"].items()}
        result["cases"][f"icp_time_c2_h{hyp}"] = r
    from icp_time import bumpy
    meshes = [bumpy(o) for o in range(8)]
    dm = icp.device_meshes(meshes, DEV)
    for name in ("lmo", "hope"):
        shape = SHAPES[name]
        Ks = torch.as_tensor(np.array(shape["K"], np.float32)).to(DEV)[None].contiguous()
        with tempfile.TemporaryDirectory() as root:
            lab, tr = make_image(root, shape, meshes, 0, np.random.default_rng(len(name)))
            d = torch.as_tensor(bop_eval.load_depth(root, "test", 1, 0, 1.0)).to(DEV)[None].contiguous()
        for hyp in (1, 5):
            n = len(lab) * hyp
            r = time_case(dm, np.repeat(lab, hyp), np.zeros(n, np.int64), perturbed(tr, hyp, rng), tr, d, Ks)
            r["ms_per_image"] = r.pop("ms")
            result["cases"][f"bop_refine_{name}_h{hyp}"] = r
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
