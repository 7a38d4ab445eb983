"""-m gpu: the IST branch from crop to pose against the fp64 evaluator of tests/ist_fp64.py, on the production path and
on trained-like weights (`realistic_trunk`: calibrated BatchNorm with near-dead channels, negative and near-zero gamma,
means several sigma off; `realistic_regressor`: relScale ~ 1, (cos, sin) away from 0).

Workload: bench.SyntheticTemplates, 2 objects x 10 templates, 6 queries and one all-zero query crop, through a
`GigaPose` model: `ResNet.forward` (the native trunk) for templates and queries, `gp_bank_write_ist` from the
channels-last view the trunk returns, `gp_ist_mlp` on the patch-major queries, RANSAC and `sort_and_pose`.  The matches
(ids, src_pts, tar_pts) are the GPU's own retrieval, which other tests prove exact.

The fp64 reference is computed from the *unfolded* module parameters, BatchNorm applied explicitly, so a mistake in the
host's fold (`ist_trunk._fold`) shows here while the folded-weight references of test_gpu_encoder_kernels.py cannot see
it.  Trunk errors are normalised per element by the magnitude of `ist_fp64.layer`.  Each bar is about 4x the largest
value measured on an H100 80GB HBM3 (700 W power limit, 1980 MHz maximum SM clock), stated next to it in brackets."""
import ctypes as C
import gc
import os
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

import ist_fp64 as I
from gigapose_b200 import _lib, ist_trunk
from gigapose_b200.engine import Engine, _ist_layout
from helpers import write_report
from test_gpu_encoder_kernels import _bank
from test_gpu_tail import BAR_MLP, BAR_POSE_R, BAR_POSE_T, pose_err, ransac_f32

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
O, T, B = 2, 10, 6
P = 256

BAR_CONV = 3e-5                 # convolutions 1-20 from the kernel's own input, of the magnitude    [7.6e-6]
BAR_OUTCONV = 1e-5              # the output convolution (1x1, fp32 rows)                           [2.5e-6]
BAR_CHAIN = 1.7e-4              # the final map from the crop against the fp64 chain                [4.2e-5]
# the regressor's own bar is test_gpu_tail.py's BAR_MLP; here the Lipschitz term of the feature difference dominates
# the bound, and the largest ratio to it was [5.6e-4] in both forms
MISLABEL_RATIO = 2              # queries read as channel-major: ratio to the regressor bound      [8.7]
MIN_DECISIONS = 200_000         # RANSAC decisions compared                                         [267 980]
MIN_UNAMBIGUOUS = 6             # hypotheses with no decision inside its margin, of 30 non-empty    [8]


def _run(model, eng, img, mask, q_obj, K, M):
    """GigaPose._retrieve_chunk step by step, keeping the query IST features and the unsorted matches."""
    tokens = model.ae_net.raw_tokens(img)
    eng.set_queries(tokens, mask, q_obj, norm_passes=2)
    m = eng.sim_topk()
    q_ist = model.ist_net.forward_by_chunk(img)
    rs, ri = eng.ist_mlp(q_ist, m)
    r = eng.ransac(m, rs, ri)
    out = eng.sort_and_pose(K, M, m, rs, ri, r)
    return out, m, q_ist, rs, ri


def _cpu(d):
    return {k: v.cpu() for k, v in d.items()}


@pytest.fixture(scope="module")
def work():
    sys.path.insert(0, ROOT)
    import bench
    with torch.no_grad():
        model = bench.build_models(DEV)
        net = model.ist_net.backbone
        net.load_state_dict(I.realistic_trunk(0))
        templates = bench.SyntheticTemplates(O, T, torch.device("cpu"))
        rgb_t = torch.cat([templates.crops(o)[0] for o in range(O)]).to(DEV)
        t_acts, t_dens = I.forward(net, rgb_t)
        t64, t_den = t_acts[-1], t_dens[-1]
        del t_acts, t_dens
        reg = I.realistic_regressor(5, t64)
        model.ist_net.regressor.load_state_dict(reg.state_dict())
        model.template_datasets = {"synthetic": templates}
        model.test_dataset_name = "synthetic"
        model.set_template_data("synthetic")
        eng = model.engines["synthetic"]
        batch, labels, _ = bench.make_queries(templates, B, seed=3)
        cat = lambda t: torch.cat([t, t[:1]]).to(DEV)
        img = torch.cat([batch.tar_img, torch.zeros_like(batch.tar_img[:1])]).to(DEV)   # + an all-zero crop
        mask, K, M = cat(batch.tar_mask), cat(batch.tar_K).float(), cat(batch.tar_M).float()
        q_obj = cat(labels - 1)
        out, m, q_ist, rs, ri = _run(model, eng, img, mask, q_obj, K, M)
        prod = model._retrieve_chunk(eng, img, mask, q_obj, K, M)
        t_ist = model.ist_net.forward_by_chunk(rgb_t)
        q_acts, q_dens = I.forward(net, img)
        torch.cuda.synchronize(DEV)
    same = all(torch.equal(out[k].view(torch.uint8), prod[k].view(torch.uint8)) for k in out)
    w = SimpleNamespace(model=model, net=net, eng=eng, reg=reg, templates=templates, img=img, q_obj=q_obj, K=K, M=M,
                        rgb_t=rgb_t, t64=t64, t_den=t_den, out=_cpu(out), m=m, q_ist=q_ist, t_ist=t_ist,
                        rs=rs, ri=ri, q_acts=q_acts, q_dens=q_dens, same_as_production=same)
    del model, net, eng, out, m, q_ist, t_ist, rs, ri, prod, q_acts, q_dens, t64, t_den
    yield w
    # the model holds reference cycles: collect it here, so that its engines' destructors and some 10 GB of fp64
    # activations do not outlive this module into later tests
    w.__dict__.clear()
    gc.collect()
    torch.cuda.synchronize(DEV)
    torch.cuda.empty_cache()


# ---------------------------------------------------------------------------------------------------- the trunk
def _dumps(trunk, x):
    d = [trunk.activation_after(x, i) for i in range(I.NUM_CONVS)]
    return d, trunk.forward(x)


def _per_layer(net, dumps, final):
    """Convolution i's output against the fp64 layer on the kernel's own input dumps, for i = 1 .. 21."""
    nchw = lambda t: t.permute(0, 3, 1, 2).double()
    acts = [nchw(dumps[0][:, 3:259, 4:260, :3])] + [nchw(t) for t in dumps[1:]]
    errs = {}
    with torch.no_grad():
        for i, s in enumerate(I.schedule(net), 1):
            ref, den = I.layer(s, acts)
            got = final if i == I.NUM_CONVS else acts[i]
            errs[i] = I.nerr(got, ref, den)
    return errs


def test_every_convolution_against_unfolded_fp64(work):
    """The production trunk engine's 21 convolutions on the seven query crops, each from the kernel's own input dump,
    against the fp64 layer with BatchNorm applied from the module's running statistics (not from the host's folded
    filters)."""
    trunk = work.net._gp_trunk_engine[1]
    dumps, final = _dumps(trunk, work.img)
    assert torch.equal(final.view(torch.int32), work.q_ist.view(torch.int32)), "the trunk is not deterministic"
    errs = _per_layer(work.net, dumps, final)
    write_report("ist_fp64_convs.json", errs)
    print("per-layer error", ["%.2e" % e for e in errs.values()])
    bad = {i: e for i, e in errs.items() if e >= (BAR_OUTCONV if i == I.NUM_CONVS else BAR_CONV)}
    assert not bad, f"convolutions over the bar: {bad}"


def test_whole_trunk_from_the_crop(work):
    """The final feature map of queries and templates, from the crops, against the fp64 chain: normalised by the final
    layer's magnitude.  Both run on the production engine through `ResNet.forward`."""
    q = I.nerr(work.q_ist, work.q_acts[-1], work.q_dens[-1])
    t = I.nerr(work.t_ist, work.t64, work.t_den)
    rel = float((work.q_ist.double() - work.q_acts[-1]).abs().max() / work.q_acts[-1].abs().max())
    write_report("ist_fp64_chain.json", {"queries": q, "templates": t, "queries_of_max": rel})
    print(f"chain: queries {q:.2e} templates {t:.2e} (of the max {rel:.2e})")
    assert work.same_as_production, "the step-by-step run differs from GigaPose._retrieve_chunk"
    assert max(q, t) < BAR_CHAIN, (q, t)


# ---------------------------------------------------------------------------------------------- the regressor
def _rows(q_feat, t_feat, q_obj, id_src, src_pts, tar_pts):
    """The regressor's input rows cat(query feature at tar_pt, template feature at src_pt) at every valid slot, in the
    order of valid.nonzero(); features [n, 256, 16, 16], templates indexed by object * T + id."""
    valid = src_pts[..., 0] != -1
    b, kk, t = valid.nonzero(as_tuple=True)
    tar, src = tar_pts[b, kk, t], src_pts[b, kk, t]
    qf = q_feat[b, :, tar[:, 1], tar[:, 0]]
    tf = t_feat[q_obj.long()[b] * T + id_src[b, kk], :, src[:, 1], src[:, 0]]
    return torch.cat([qf, tf], 1), valid


def _regressor_check(work, m, rs, ri, form):
    """Every valid slot's outputs against the fp64 regressor on the fp64 features: the largest ratio of the error to
    BAR_MLP[form] * magnitude + lipschitz(|GPU features - fp64 features|), and the features' own error."""
    m = {k: v.to(DEV) for k, v in m.items()}
    args = (work.q_obj, m["id_src"], m["src_pts"], m["tar_pts"])
    rows, valid = _rows(work.q_ist.double(), work.t_ist.double(), *args)
    rows64, _ = _rows(work.q_acts[-1], work.t64, *args)
    den_rows, _ = _rows(work.q_dens[-1], work.t_den, *args)
    feat = I.nerr(rows, rows64, den_rows)
    (s64, sden), (i64, iden) = I.regressor(work.reg, rows64)
    ls, li = I.lipschitz(work.reg, (rows - rows64).abs())
    es = (rs[valid].double() - s64[:, 0]).abs() / (BAR_MLP[form] * sden[:, 0] + ls[:, 0])
    ei = (ri[valid].double() - i64).abs() / (BAR_MLP[form] * iden + li)
    invalid_ok = bool((rs[~valid] == -1000).all()) and bool((ri[~valid] == -1000).all())
    return dict(rows=int(valid.sum()), ratio=float(max(es.max(), ei.max())), features=feat,
                lipschitz_scale_max=float(ls.max()), err_scale_max=float((rs[valid].double() - s64[:, 0]).abs().max()),
                relScale_range=[float(s64.min()), float(s64.max())], invalid_slots_minus_1000=invalid_ok)


def _tc_outputs(work, monkeypatch, q_ist, m):
    """The tensor-core form (GIGAPOSE_MLP_SIMT=0) on an engine holding the same IST bank."""
    monkeypatch.setenv("GIGAPOSE_MLP_SIMT", "0")
    eng = Engine(O, T, len(q_ist), device=DEV, k=work.eng.k)
    for o in range(O):
        eng.bank_write_ist(o, 0, work.t_ist[o * T:(o + 1) * T])
    eng.set_ist_weights(work.model.ist_net.regressor)
    eng.set_queries(torch.zeros(len(q_ist), P, 1024), torch.ones(len(q_ist), 16, 16), work.q_obj, norm_passes=0)
    rs, ri = eng.ist_mlp(q_ist, m)
    torch.cuda.synchronize(DEV)
    return rs, ri


def test_bank_and_query_layouts(work):
    """The template IST bank holds the trunk's output bit for bit (a memcpy of the channels-last view); the queries are
    passed as patch-major, and the same buffer mislabelled as channel-major misses the regressor bound (by 8.7x, and
    by 1.6e4x the ratio of the right layout; the bound's Lipschitz term is loose, see below)."""
    eng = work.eng
    bank = _bank(eng)["ist"].view(torch.float32).view(O * T, P, 256)
    assert torch.equal(bank.view(torch.int32), work.t_ist.permute(0, 2, 3, 1).reshape(O * T, P, 256).view(torch.int32))
    assert _ist_layout(work.q_ist)[1] == _lib.LAYOUT_PATCH_MAJOR
    m = work.m
    n = len(work.q_ist)
    rs, ri = torch.empty(n, eng.k, P, device=DEV), torch.empty(n, eng.k, P, 2, device=DEV)
    _lib.check(eng.lib.gp_ist_mlp(eng._h, 0, n, work.q_ist.data_ptr(), _lib.LAYOUT_CHANNEL_MAJOR,
                                  C.byref(eng._matches_struct(m)), rs.data_ptr(), ri.data_ptr(), eng.stream))
    torch.cuda.synchronize(DEV)
    bad = _regressor_check(work, m, rs, ri, "simt")
    good = _regressor_check(work, m, work.rs, work.ri, "simt")
    write_report("ist_fp64_mislabelled.json", {"patch_major": good["ratio"], "channel_major": bad["ratio"]})
    assert good["ratio"] < 1 and bad["ratio"] > MISLABEL_RATIO and bad["ratio"] > 1e3 * good["ratio"], \
        (good["ratio"], bad["ratio"])


def _outputs64(work, m, form):
    """At every slot of the matches m (CPU tensors): the fp64 regressor's outputs on the fp64 features, and the bound
    BAR_MLP[form] * magnitude + lipschitz(|GPU features - fp64 features|); -1000 and 0 at invalid slots."""
    args = (work.q_obj, m["id_src"].to(DEV), m["src_pts"].to(DEV), m["tar_pts"].to(DEV))
    rows64, valid = _rows(work.q_acts[-1], work.t64, *args)
    rows, _ = _rows(work.q_ist.double(), work.t_ist.double(), *args)
    (s64, sden), (i64, iden) = I.regressor(work.reg, rows64)
    ls, li = I.lipschitz(work.reg, (rows - rows64).abs())
    n, k = m["id_src"].shape
    sc64, lsc = torch.full((n, k, P), -1000.0, dtype=torch.float64), torch.zeros(n, k, P, dtype=torch.float64)
    cs64, lcs = torch.full((n, k, P, 2), -1000.0, dtype=torch.float64), torch.zeros(n, k, P, 2, dtype=torch.float64)
    valid = valid.cpu()
    sc64[valid], cs64[valid] = s64[:, 0].cpu(), i64.cpu()
    lsc[valid], lcs[valid] = (BAR_MLP[form] * sden[:, 0] + ls[:, 0]).cpu(), (BAR_MLP[form] * iden + li).cpu()
    return sc64.numpy(), cs64.numpy(), lsc.numpy(), lcs.numpy()


def _decisions_against_fp64(src, tar, sc, cs, sc64, cs64, lsc=None, lcs=None):
    """RANSAC decisions of the fp32 restatement (`ransac_f32`, which the kernel equals bit for bit) on the GPU's outputs
    against fp64 decisions on fp64's, over [N, 256] hypotheses.  The margin takes the measured output difference;
    every decision outside it must be equal.  With lsc / lcs the decisions inside the margin those bounds would give
    are counted as well."""
    N = src.shape[0]
    want, detail = ransac_f32(src, tar, sc.astype(np.float32), cs.astype(np.float32), 14.0, 14)
    d_sc, d_cs = np.abs(sc - sc64), np.abs(cs - cs64)
    rep = dict(hypotheses=N, empty_hypotheses=0, decisions=0, ambiguous_decisions=0, ambiguous_hypotheses=0)
    if lsc is not None:
        rep.update(ambiguous_decisions_lipschitz=0, ambiguous_hypotheses_lipschitz=0)
    fp64 = []
    for i in range(N):
        r = I.ransac(src[i], tar[i], sc64[i], cs64[i], d_sc=d_sc[i], d_cs=d_cs[i])
        fp64.append(r)
        if detail[i] is None:
            rep["empty_hypotheses"] += 1
            assert r.D is None
            continue
        keep, inl = detail[i]
        off = ~np.eye(len(keep), dtype=bool)
        bad = (inl != r.D) & ~r.near & off
        assert not bad.any(), f"hypothesis {i}: {int(bad.sum())} decisions differ from fp64 outside the margin"
        rep["decisions"] += int(off.sum())
        rep["ambiguous_decisions"] += int(r.near.sum())
        rep["ambiguous_hypotheses"] += int(r.near.any())
        if lsc is not None:
            near = I.ransac(src[i], tar[i], sc64[i], cs64[i], d_sc=lsc[i], d_cs=lcs[i]).near
            rep["ambiguous_decisions_lipschitz"] += int(near.sum())
            rep["ambiguous_hypotheses_lipschitz"] += int(near.any())
    return rep, want, detail, fp64


@pytest.mark.parametrize("form", ["simt", "tc"])
def test_regressor_against_fp64_on_fp64_features(work, form, monkeypatch):
    """gp_ist_mlp's outputs at every valid slot of the production matches, against the fp64 regressor on the fp64
    features: |out - out64| <= BAR_MLP[form] * magnitude + lipschitz(delta), delta the measured difference between the
    GPU's features and fp64's.  The Lipschitz term is rigorous but loose (it assumes every sign lines up), so the
    features themselves must also be within BAR_CHAIN of fp64: a trunk that is wrong by more cannot hide behind it.
    Both forms' RANSAC decisions (ransac_f32 on their outputs) must equal fp64's outside the margin of
    test_ransac_decisions_against_fp64; how many decisions and winning inlier sets the tensor-core form changes against
    the SIMT form is reported: the decision-level measure DESIGN.md section 8 item 2 asks for."""
    rs, ri = (work.rs, work.ri) if form == "simt" else _tc_outputs(work, monkeypatch, work.q_ist, work.m)
    rep = _regressor_check(work, work.m, rs, ri, form)
    m = _cpu(work.m)
    N = m["id_src"].numel()
    sc64, cs64, _, _ = _outputs64(work, m, form)
    flat = lambda a, *s: a.reshape(N, P, *s)
    pts = (flat(m["src_pts"].numpy(), 2), flat(m["tar_pts"].numpy(), 2))
    dec, want, _, _ = _decisions_against_fp64(*pts, flat(rs.cpu().numpy(), ).astype(np.float64),
                                              flat(ri.cpu().numpy(), 2).astype(np.float64), flat(sc64), flat(cs64, 2))
    rep["ransac"] = dec
    if form == "tc":
        simt, sd = ransac_f32(*pts, flat(work.rs.cpu().numpy()), flat(work.ri.cpu().numpy(), 2), 14.0, 14)
        _, td = ransac_f32(*pts, flat(rs.cpu().numpy()), flat(ri.cpu().numpy(), 2), 14.0, 14)
        rep["decisions_other_than_simt"] = sum(int((a[1] != b[1]).sum()) for a, b in zip(sd, td) if a is not None)
        rep["inlier_sets_other_than_simt"] = int((simt["in_src"] != want["in_src"]).any(axis=(1, 2)).sum())
    write_report(f"ist_fp64_regressor_{form}.json", rep)
    print(form, rep)
    assert rep["invalid_slots_minus_1000"]
    assert rep["rows"] > 1000, rep["rows"]
    assert rep["features"] < BAR_CHAIN, rep
    assert rep["ratio"] < 1, rep


# -------------------------------------------------------------------------------------------------------- RANSAC
def test_ransac_decisions_against_fp64(work):
    """RANSAC on the production outputs against fp64 RANSAC on the fp64 regressor outputs, per (query, hypothesis) of
    the sorted predictions.  The kernel's M, inlier points and idx_failed are those of `ransac_f32` (its bit-exact
    restatement), so its decisions are the restatement's.  A decision's margin is 2^-18 of its coordinates' magnitudes
    plus the move of the proposer's similarity under the *measured* difference between the GPU's and fp64's regressor
    outputs (ist_fp64.decisions).  The rigorous bound of test_regressor_against_fp64_on_fp64_features is ~1e3 x looser
    (its Lipschitz term assumes every sign lines up); the decisions and hypotheses it would leave ambiguous are
    reported, not asserted.
    - every decision outside its margin equals fp64;
    - a hypothesis none of whose decisions lies inside a margin has fp64's winner, inlier set, idx_failed and count;
      its M is fp64's within the product rule's bound on the measured output difference (which a single dominant term
      meets with equality: the 2 x 2 block measures ~1) plus fp32 rounding;
    - every pose is fp64 pose lifting of the kernel's M within test_gpu_tail.py's bars.
    MIN_DECISIONS and MIN_UNAMBIGUOUS are fixed floors under what this workload gives, so the test cannot pass
    vacuously."""
    out = work.out
    n, k = out["id_src"].shape
    N = n * k
    sc64, cs64, lsc, lcs = _outputs64(work, out, "simt")
    flat = lambda a, *s: a.reshape(N, P, *s)
    src, tar = flat(out["src_pts"].numpy(), 2), flat(out["tar_pts"].numpy(), 2)
    sc, cs = flat(out["relScale"].numpy()).astype(np.float64), flat(out["relInplane"].numpy(), 2).astype(np.float64)
    sc64, cs64 = flat(sc64), flat(cs64, 2)
    rep, want, detail, fp64 = _decisions_against_fp64(src, tar, sc, cs, sc64, cs64, flat(lsc), flat(lcs, 2))
    Mk = out["M"].numpy().reshape(N, 3, 3)
    assert np.array_equal(Mk.view(np.int32), want["M"].view(np.int32))
    assert np.array_equal(flat(out["ransac_src_pts"].numpy(), 2), want["in_src"])
    assert np.array_equal(out["idx_failed"].numpy().reshape(N), want["failed"].astype(bool))
    rep.update(unambiguous_hypotheses=0, M_ratio_rotation=0.0, M_ratio_translation=0.0)
    for i, r in enumerate(fp64):
        if detail[i] is None or r.near.any():
            continue
        rep["unambiguous_hypotheses"] += 1
        b, h = divmod(i, k)
        keep, inl = detail[i]
        best = int(np.argmax(inl.sum(1)))
        assert best == r.best, (b, h, best, r.best)
        assert np.array_equal(out["ransac_src_pts"][b, h].numpy(), r.in_src), (b, h)
        assert np.array_equal(out["ransac_tar_pts"][b, h].numpy(), r.in_tar), (b, h)
        assert bool(out["idx_failed"][b, h]) == r.failed and int(out["ransac_scores"][b, h].sum()) == r.count, (b, h)
        j = keep[best]
        c, s, kk = cs64[i, j, 0], cs64[i, j, 1], sc64[i, j]
        dsc, dc, ds = abs(sc[i, j] - kk), abs(cs[i, j, 0] - c), abs(cs[i, j, 1] - s)
        dA = abs(c) * dsc + abs(kk) * dc + dsc * dc
        dB = abs(s) * dsc + abs(kk) * ds + dsc * ds
        sj = src[i, j].astype(np.float64) * 14
        mag = np.abs(r.M[:2, :2]) @ np.abs(sj) + np.abs(tar[i, j] * 14.0)
        lim_r = np.array([[dA, dB], [dB, dA]]) + 2.0 ** -22 * np.abs(r.M[:2, :2])
        lim_t = np.hypot(dA, dB) * np.hypot(*sj) + 2.0 ** -18 * mag
        rep["M_ratio_rotation"] = max(rep["M_ratio_rotation"], float((np.abs(Mk[i, :2, :2] - r.M[:2, :2]) / lim_r).max()))
        rep["M_ratio_translation"] = max(rep["M_ratio_translation"], float((np.abs(Mk[i, :2, 2] - r.M[:2, 2]) / lim_t).max()))
    templates = work.templates
    tK, tM = templates.K.expand(O, 3, 3), templates.M
    tP = templates.poses[None].expand(O, T, 4, 4)
    ref = I.pose(work.q_obj.cpu(), work.K.cpu(), work.M.cpu(), out["id_src"], out["M"], tK, tM, tP)
    eR, eT, bottom = pose_err(out["pred_poses"], ref)
    rep.update(pose_R=eR, pose_t=eT)
    write_report("ist_fp64_ransac.json", rep)
    print("RANSAC", rep)
    assert rep["M_ratio_rotation"] <= 1 and rep["M_ratio_translation"] <= 1, rep
    assert bottom and eR < BAR_POSE_R and eT < BAR_POSE_T, rep
    assert rep["decisions"] >= MIN_DECISIONS and rep["unambiguous_hypotheses"] >= MIN_UNAMBIGUOUS, rep


# ---------------------------------------------------------------------------------------------- negative controls
@pytest.mark.parametrize("name", list(I.MUTATED_FOLDS))
def test_mutated_folds_miss_by_far(work, name, monkeypatch):
    """`ist_trunk._fold` replaced by a wrong fold (eps dropped, 1e-6 or 1e-3, or the bias without 1 / sqrt(var + eps)):
    a trunk built with it misses the per-layer bar by >= 10x on every BatchNorm layer (each carries planted near-dead
    channels), and its features miss the feature bound of the regressor test by >= 10x."""
    monkeypatch.setattr(ist_trunk, "_fold", I.MUTATED_FOLDS[name])
    x = work.img[[0, B]]                              # one query and the zero crop
    trunk = ist_trunk.NativeISTTrunk(work.net, DEV, max_crops=len(work.img))
    dumps, final = _dumps(trunk, x)
    errs = _per_layer(work.net, dumps, final)
    q_ist = trunk.forward(work.img)
    t_ist = trunk.forward(work.rgb_t)
    torch.cuda.synchronize(DEV)
    mut = SimpleNamespace(**{**vars(work), "q_ist": q_ist, "t_ist": t_ist})
    rep = _regressor_check(mut, work.m, work.rs, work.ri, "simt")
    write_report(f"ist_fp64_control_{name.replace(' ', '_')}.json", {"per_layer": errs, "features": rep["features"]})
    print(name, "per-layer min %.2e" % min(list(errs.values())[:20]), "features %.2e" % rep["features"])
    weak = {i: e for i, e in errs.items() if i < I.NUM_CONVS and e < 10 * BAR_CONV}
    assert not weak, f"{name}: layers within 10x the bar: {weak}"
    assert rep["features"] > 10 * BAR_CHAIN, rep["features"]
