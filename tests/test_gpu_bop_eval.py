"""Row f7 on the GPU: gp_render_depth against the one-sample port (oracle/bop_port.render_depth), gp_bop_vsd and gp_bop_mssd_mspd against
the fp32 port bit for bit and against the fp64 definitions, and evaluate() end to end on a synthetic BOP tree.  The
launch counter around evaluate() is checked in tests/test_gpu_z_bop_launch_count.py."""
import json

import numpy as np
import pytest
import torch

from bop_tree import rot, spheroid, tetra, write_tree
from gigapose_b200 import _lib, bop_eval, icp
from icp_scenes import T_ASM, T_ELL, assembly, ellipsoid, perturb, plate, pose
from oracle import bop_port

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
H, W = 117, 203                                  # not a multiple of the 256-thread tiles
KS = [np.array([[300.0, 0, 101.3], [0, 302.0, 57.9], [0, 0, 1]], np.float32),
      np.array([[280.0, 0, 95.0], [0, 281.0, 61.0], [0, 0, 1]], np.float32)]


def _report(name, obj):
    """The measured agreement, for DESIGN.md §3 (shown with pytest -s)."""
    print(name, json.dumps(obj))


def _gpu_render(mesh, poses, K, z_near=10.0):
    dm = icp.device_meshes([mesh], DEV)[0]
    poses = torch.as_tensor(np.asarray(poses, np.float32), device=DEV).reshape(-1, 4, 4).contiguous()
    n = poses.shape[0]
    ws = torch.empty(n * H * W * 8, dtype=torch.uint8, device=DEV)
    d = torch.empty(n, H, W, device=DEV)
    b = torch.empty(n, 4, dtype=torch.int64, device=DEV)
    bop_eval.render_depth(dm, poses, torch.as_tensor(K, device=DEV).contiguous(), H, W, z_near, ws, d, b)
    return d.cpu().numpy(), b.cpu().numpy()


def _cases():
    ell, asm, pl = ellipsoid(), assembly(), plate()
    T_PL = pose(rot([1, 0.2, 0], 30), [5.0, 3.0, 600.0])
    half_out = T_ELL.copy()
    half_out[0, 3] = 230.0                       # partly outside the image
    behind = T_ELL.copy()
    behind[2, 3] = -200.0                        # every vertex at z <= z_near: an empty render
    return [(ell, [T_ELL, perturb(T_ELL, [0, 1, 0], 8, [6, -4, 10]), half_out, behind]),
            (asm, [T_ASM, perturb(T_ASM, [1, 0, 0], 5, [0, 3, -8])]), (pl, [T_PL])]


def test_render_depth_is_bit_identical_to_the_one_sample_port():
    for mesh, poses in _cases():
        for K in KS:
            d, b = _gpu_render(mesh, poses, K)
            for i, T in enumerate(poses):
                want = bop_port.render_depth(mesh["vertices"], mesh["faces"], T, K, H, W, 10.0)
                np.testing.assert_array_equal(d[i].view(np.uint32), want["depth"].view(np.uint32))
                np.testing.assert_array_equal(b[i], want["box"])
    empty = _gpu_render(_cases()[0][0], [_cases()[0][1][3]], KS[0])
    assert not empty[0].any() and empty[1][0].tolist() == [0, 0, W, H]


def _scene(frame):
    """Measured depth of frame 0 / 1: the ellipsoid or the assembly in front of a background plane, 5 % missing
    pixels and a box occluder over part of the object."""
    K = KS[frame]
    mesh, T = (ellipsoid(), T_ELL) if frame == 0 else (assembly(), T_ASM)
    obj = bop_port.render_depth(mesh["vertices"], mesh["faces"], T, K, H, W, 10.0)["depth"]
    z = float(T[2, 3]) + 150.0
    bg = np.full((H, W), z, np.float32)
    d = np.where(obj > 0, obj, bg)
    rng = np.random.default_rng(frame)
    d[rng.random((H, W)) < 0.05] = 0
    ys, xs = np.nonzero(obj)
    d[ys.min():ys.max() + 1, xs.min():(xs.min() + xs.max()) // 2] = float(T[2, 3]) - 100.0
    d[:ys.min() + 3] = np.where(obj[:ys.min() + 3] > 0, d[:ys.min() + 3], 0)
    return d.astype(np.float32)


def test_vsd_counts_are_bit_identical_to_the_fp32_port():
    taus = bop_eval.TAUS
    depth_test = np.stack([_scene(0), _scene(1)])
    renders, boxes, pairs, diam = [], [], [], []     # pairs: (frame, est render, gt render)
    for f, (mesh, T, d) in enumerate([(ellipsoid(), T_ELL, 180.0), (assembly(), T_ASM, 110.0)]):
        half_out = T.copy()
        half_out[0, 3] += 200.0
        behind = T.copy()
        behind[2, 3] = -200.0
        ests = [T, perturb(T, [0, 1, 0], 4, [3, -2, 5]), perturb(T, [1, 0, 1], 15, [0, 0, 30]), half_out, behind]
        dd, bb = _gpu_render(mesh, [T] + ests, KS[f])
        base = len(renders)
        renders += list(dd)
        boxes += list(bb)
        pairs += [(f, base + 1 + i, base) for i in range(len(ests))]
        diam += [d] * len(ests)
    pairs = np.array(pairs, np.int32)
    t = lambda a, dt=None: torch.as_tensor(np.ascontiguousarray(a, dt), device=DEV)
    counts, errors = bop_eval.vsd(t(depth_test), t(np.stack(KS)), t(pairs[:, 0]), t(np.stack(renders)), t(np.stack(boxes)),
                                  t(pairs[:, 1]), t(np.stack(renders)), t(np.stack(boxes)), t(pairs[:, 2]),
                                  t(diam, np.float32), 15.0, taus)
    counts, errors = counts.cpu().numpy(), errors.cpu().numpy()
    decisions = 0
    for p, (f, e, g) in enumerate(pairs):
        c32, e32 = bop_port.vsd_fp32(depth_test[f], KS[f], renders[e], boxes[e], renders[g], boxes[g], diam[p], 15.0, taus)
        np.testing.assert_array_equal(counts[p], c32)
        np.testing.assert_array_equal(errors[p].view(np.uint32), e32.view(np.uint32))
        c64, e64 = bop_port.vsd_fp64(depth_test[f], KS[f], renders[e], renders[g], diam[p], 15.0, taus)
        decisions += int(np.abs(c64 - c32).sum())
        assert np.abs(e64 - e32).max() <= max(1e-6, 4.0 * np.abs(c64 - c32).sum() / max(c64[1], 1)) + 1e-6
    assert counts[0, 0] == counts[0, 1] and not errors[0].any()          # estimate == ground truth
    assert counts[4, 1] > 0 and counts[4, 0] == 0 and np.all(errors[4] == 1)   # empty estimate: union = visible gt
    _report("vsd decisions", dict(pairs=len(pairs), pixels_in_unions=int(counts[:, 1].sum()),
                                           fp32_vs_fp64_count_differences=decisions))
    assert decisions <= 1e-3 * counts[:, 1].sum()


def test_mssd_mspd_bit_identical_to_the_fp32_port_and_bounded_by_fp64():
    tV, _ = tetra(60.0)
    sV, _ = spheroid(40.0, 25.0)
    step = np.eye(4)
    step[:3, :3] = rot([0, 0, 1], 360.0 / 96)
    disc = [np.linalg.matrix_power(step, k) for k in range(1, 96)]
    sym_t = bop_eval.symmetry_transforms({})
    sym_d = bop_eval.symmetry_transforms(dict(symmetries_discrete=disc))
    sym_c = bop_eval.symmetry_transforms(dict(symmetries_continuous=[(np.array([0, 0, 1.0]), np.zeros(3))]))
    objs = [(tV, sym_t), (sV, sym_d), (sV, sym_c)]
    Tg = pose(rot([0.4, 1, 0.1], 25), [10.0, -5.0, 650.0])
    cases = []                                         # (object, frame, pose_est, pose_gt)
    cases += [(0, 0, perturb(Tg, [1, 1, 0], 3, [2, 1, -4]), Tg), (0, 1, Tg, Tg)]
    one_step = pose(Tg[:3, :3].astype(np.float64) @ step[:3, :3], Tg[:3, 3])
    cases += [(1, 0, one_step, Tg), (1, 1, perturb(Tg, [0, 1, 0], 6, [0, 0, 5]), Tg)]
    cont = pose(Tg[:3, :3].astype(np.float64) @ rot([0, 0, 1], 37.3), Tg[:3, 3])
    cases += [(2, 0, cont, Tg), (2, 1, perturb(cont, [1, 0, 0], 2, [1, 1, 1]), Tg)]
    vo = np.cumsum([0] + [len(v) for v, _ in objs]).astype(np.int32)
    so = np.cumsum([0] + [len(s) for _, s in objs]).astype(np.int32)
    t = lambda a, dt=np.float32: torch.as_tensor(np.ascontiguousarray(a, dt), device=DEV)
    mssd, mspd = bop_eval.mssd_mspd(t([c[0] for c in cases], np.int32), vo.tolist(), t(np.concatenate([v for v, _ in objs])),
                                    so.tolist(), t(np.concatenate([s for _, s in objs])), t(np.stack(KS)),
                                    t([c[1] for c in cases], np.int32), t(np.stack([c[2] for c in cases])),
                                    t(np.stack([c[3] for c in cases])))
    mssd, mspd = mssd.cpu().numpy(), mspd.cpu().numpy()
    worst = 0.0
    for p, (o, f, Pe, Pg) in enumerate(cases):
        V, S = objs[o]
        m32 = bop_port.mssd_mspd_fp32(V, S.astype(np.float32), Pe, Pg, KS[f])
        assert mssd[p].view(np.uint32) == np.float32(m32[0]).view(np.uint32), p
        assert mspd[p].view(np.uint32) == np.float32(m32[1]).view(np.uint32), p
        m64 = bop_port.mssd_mspd_fp64(V, S.astype(np.float32), Pe.astype(np.float32), Pg.astype(np.float32), KS[f])
        worst = max(worst, abs(m64[0] - mssd[p]) / 700.0, abs(m64[1] - mspd[p]) / 300.0)
    assert worst < 2e-6, worst                         # relative to |t| and to f: fp32 rounding of the transforms
    chord = 2 * 40.0 * np.sin(np.pi / 96)
    assert mssd[2] < 1e-3 < chord                      # one declared step: fp32 rounding, not the chord
    assert mssd[4] <= 40.0 * np.pi / 315 + 1e-3       # continuous: within half a discretisation step
    assert mssd[1] < 1e-3 and mspd[1] < 1e-3           # identical poses
    _report("mssd / mspd vs fp64", dict(worst_relative=worst, one_step_mssd=float(mssd[2]), chord=chord,
                                       continuous_mssd=float(mssd[4]), half_step_bound=40.0 * np.pi / 315))


def _tree(root):
    """Two scenes, three objects (one with a declared discrete symmetry), repeated instances, perturbed estimates."""
    Hs, Ws = 96, 128
    Ks = [np.array([[150.0, 0, 63.0], [0, 150.0, 47.0], [0, 0, 1]]), np.array([[140.0, 0, 65.0], [0, 141.0, 49.0], [0, 0, 1]])]
    models = {1: tetra(60.0), 2: spheroid(40.0, 25.0, n_lat=10, n_lon=24), 3: (assembly()["vertices"], assembly()["faces"])}
    flip = np.diag([-1.0, -1, 1, 1])
    info = {1: dict(diameter=84.9), 2: dict(diameter=80.0, symmetries_discrete=[flip.ravel().tolist()]),
            3: dict(diameter=110.0)}
    rng = np.random.default_rng(7)
    scenes, targets, results = {}, [], []
    for s in (1, 2):
        scenes[s] = {}
        for im in range(2):
            K = Ks[(s + im) % 2]
            gts = [(1, rot([0, 1, 0], 20 * im + 5 * s), [-60.0, 0, 650.0]), (2, rot([1, 0, 0], 30), [50.0, -30.0, 700.0]),
                   (2, rot([0, 1, 1], 50), [40.0, 60.0, 800.0]), (3, rot([1, 1, 0], 40), [0.0, 10.0, 900.0])]
            depth = np.full((Hs, Ws), 1500.0, np.float32)
            for o, R, t in gts:
                T = pose(R, t)
                d = bop_port.render_depth(models[o][0], models[o][1], T, K, Hs, Ws, 10.0)["depth"]
                depth = np.where((d > 0) & (d < depth), d, depth)
            depth[rng.random((Hs, Ws)) < 0.03] = 0
            png = np.round(depth / 0.1).astype(np.uint16)
            scenes[s][im] = dict(gt=gts, visib=[0.8, 0.9, 0.05 if im == 0 else 0.6, 0.7], K=K, depth_scale=0.1, png=png)
            targets += [(s, im, 1, 1), (s, im, 2, 2 if im else 1), (s, im, 3, 1)]
            for k, (o, R, t) in enumerate(gts):
                for rep in range(2):
                    dR = rot(rng.normal(size=3), rng.uniform(0, 12))
                    dt = rng.normal(size=3) * [4, 4, 15] * (rep + 1)
                    if o == 2 and rep == 0 and k == 1:       # the ground truth turned by its declared symmetry
                        dR, dt = R @ flip[:3, :3] @ R.T, np.zeros(3)
                    results.append(dict(scene_id=s, im_id=im, obj_id=o, score=float(rng.random()), R=dR @ R,
                                        t=(np.asarray(t) + dt).reshape(3, 1), time=0.1 * (s + im)))
    write_tree(str(root), models, info, scenes, targets)
    return results, models, info, scenes


def _port_errors(setup, errors, models):
    """The port's per-pair errors from its one-sample depth renders and the kernels' fp32 arithmetic."""
    res, groups, scenes = setup["results"], setup["groups"], setup["scenes"]
    out = dict(vsd=[], mssd=[], mspd=[])
    for p in range(len(errors["group"])):
        g = groups[int(errors["group"][p])]
        s, im, o = g["scene_id"], g["im_id"], g["obj_id"]
        K = scenes[s]["K"][im].astype(np.float32)
        d_test = bop_eval.load_depth(setup["dataset_dir"], "test", s, im, scenes[s]["depth_scale"][im])
        e = res[int(errors["est"][p])]
        gt = scenes[s]["gt"][im][int(errors["gt"][p])]
        Pe, Pg = bop_eval._pose(e["R"], e["t"]).astype(np.float32), bop_eval._pose(gt["R"], gt["t"]).astype(np.float32)
        V, F = models[o]
        re = bop_port.render_depth(V, F, Pe, K, *d_test.shape, 10.0)
        rg = bop_port.render_depth(V, F, Pg, K, *d_test.shape, 10.0)
        _, e32 = bop_port.vsd_fp32(d_test, K, re["depth"], re["box"], rg["depth"], rg["box"],
                                   np.float32(setup["info"][o]["diameter"]), 15.0, bop_eval.TAUS)
        m = bop_port.mssd_mspd_fp32(V, bop_eval.symmetry_transforms(setup["info"][o]).astype(np.float32), Pe, Pg, K)
        out["vsd"].append(e32)
        out["mssd"].append(m[0])
        out["mspd"].append(m[1])
    return {k: np.array(v) for k, v in out.items()}


def test_evaluate_end_to_end_matches_the_port(tmp_path):
    results, models, info, scenes = _tree(tmp_path)
    out = bop_eval.evaluate(results, str(tmp_path), out_dir=str(tmp_path / "eval"), device=DEV)
    setup = bop_eval.prepare(results, str(tmp_path))
    err = out["errors"]
    assert len(err["group"]) == sum(len(g["est"]) * len(g["gt"]) for g in setup["groups"]) >= 16
    port = _port_errors(setup, err, models)
    np.testing.assert_array_equal(err["vsd"].view(np.uint32), port["vsd"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(err["mssd"].view(np.uint32), port["mssd"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(err["mspd"].view(np.uint32), port["mspd"].astype(np.float32).view(np.uint32))
    assert (err["mssd"] < 1e-3).any()                  # the flipped estimate of the symmetric object
    # the port's matcher on the GPU's errors gives exactly the same recalls
    rank = [{e: i for i, e in enumerate(g["est"])} for g in setup["groups"]]
    pairs = [dict(target=int(err["group"][p]), rank=rank[int(err["group"][p])][int(err["est"][p])], gt=int(err["gt"][p]),
                  vsd=err["vsd"][p], mssd=err["mssd"][p], mspd=err["mspd"][p]) for p in range(len(err["group"]))]
    targets = [dict(valid=dict(zip(g["gt"], g["valid"].tolist())), diameter=info[g["obj_id"]]["diameter"])
               for g in setup["groups"]]
    ref = bop_port.average_recalls(pairs, targets, bop_eval.TAUS, bop_eval.THETA_VSD, bop_eval.THETA_MSSD,
                                   bop_eval.THETA_MSPD, 128 / 640)
    for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd"):
        assert out[k] == ref[k], k
    np.testing.assert_array_equal(out["recall_vsd"], ref["recall_vsd"])
    assert out["n_targets"] == sum(1 for t in targets for v in t["valid"].values() if v)
    assert 0 < out["ar"] < 1
    scores = json.load(open(tmp_path / "eval" / "scores_bop19.json"))
    assert scores["bop19_average_recall"] == out["ar"]
    assert scores["bop19_average_time_per_image"] == pytest.approx(np.mean([0.1, 0.2, 0.2, 0.3]))
    _report("end to end", {k: out[k] for k in ("ar", "ar_vsd", "ar_mssd", "ar_mspd", "n_targets")})

