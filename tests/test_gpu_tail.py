"""-m gpu: the kernels after the similarity search -- top-k select and merge, the IST regressor, RANSAC, re-sort and pose
lifting -- each alone against an exact or fp64 statement of the same operation, with inputs planted where these kernels
decide: exact score ties inside a thread, across lanes, warps and shards, inlier distances of exactly the threshold,
equal RANSAC scores in different warps, invalid slots at both ends of a crop, windows of a batch.

Caller-made inputs go through the public C ABI; outputs are prefilled with sentinels, so a slot a kernel forgets to
write cannot pass.  Integer outputs and copies are compared bit for bit.  Float bars are about 4x the largest value
measured on an H100 SXM (80 GB, 400 W power limit), stated next to each bar."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from gigapose_b200 import _lib, synth
from gigapose_b200._lib import check
from gigapose_b200.engine import Engine
from oracle import port

from helpers import engine_from_case, write_report

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)
P = 256
PAD_ID = 0x7FFFFFFF
SENT = -7                         # integer sentinel
# --- bars, with the largest value measured on an H100 SXM (400 W limit) in brackets
BAR_MLP = {"simt": 1.5e-9, "tc": 8e-9}  # regressor outputs, |out - out64| / propagated magnitude  [3.3e-10, 1.9e-9]
BAR_POSE_R = 3.5e-7                     # pose lifting, rotation, absolute                         [8.3e-8]
BAR_POSE_T = 3.5e-4                     # pose lifting, translation, relative to max(|t|, 1)       [8.4e-5]
# per-patch and per-template scores of the winners against the fp32 oracle.  The split product drops lo * lo (2^-18 of
# sum |q||t|), so the planted templates equal to the query (similarity 1) sit furthest off: score_pts [8.8e-6],
# score_src [4.1e-6]
BAR_SCORE_PTS = 3.5e-5


def _stream():
    return torch.cuda.current_stream(DEV).cuda_stream


def _lib_():
    return _lib.load()


def nan_f32(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def sent_i64(*shape):
    return torch.full(shape, SENT, dtype=torch.int64, device=DEV)


def bits(t):
    return t.contiguous().view(torch.int32)


def _matches_struct(m):
    return _lib.GpMatches(*(m[k].data_ptr() for k in ("id_src", "score_src", "score_pts", "tar_pts", "src_pts")))


def sentinel_matches(B, k):
    return dict(id_src=sent_i64(B, k), score_src=nan_f32(B, k), score_pts=nan_f32(B, k, P),
                tar_pts=sent_i64(B, k, P, 2), src_pts=sent_i64(B, k, P, 2))


def pts_of(valid, idx):
    """(x, y) = (idx % 16, idx // 16) where valid, else (-1, -1)."""
    idx = torch.as_tensor(idx, dtype=torch.int64)
    valid = torch.as_tensor(valid, dtype=torch.bool)
    xy = torch.stack([idx % 16, idx // 16], -1)
    return torch.where(valid[..., None], xy, torch.full_like(xy, -1))


def python_topk(scores, ids, k):
    """Positions of the k winners: score descending, then id ascending, then position (the kernels' order)."""
    return sorted(range(len(scores)), key=lambda c: (-scores[c], ids[c], c))[:k]


# ========================================================================================================= top-k select
G0 = [1, 3, 9, 100, 200, 259, 515, 771]  # copies of the best template: 9 = another lane of 3's warp, 100 / 200 = other
G1 = [20, 50, 276, 532]                  # warps, 259 / 515 / 771 = 3's own thread (256 apart); copies of the second best
GAP = 1e-5                               # distinct oracle scores near the top-k are at least this far apart

# (T, k, B): T = k, the edges of one 256-template pass and several templates per thread; B = 3 adds a second object and
# a fully masked query; T = 1000 keeps B = 1 (the reference layout is ~1 GB per query on the host)
TOPK_CASES = [(5, 5, 2), (255, 32, 2), (256, 5, 2), (257, 32, 3), (257, 1, 2), (576, 5, 1), (1000, 32, 1)]


def _planted_topk_case(T, B, seed):
    """Per object, template src0 is the first query's own descriptors (the clear winner) and src1 a noisy copy of them
    (the runner-up); identical copies of src0 go to the ids in G0 and of src1 to those in G1."""
    O = 2 if B == 3 else 1
    labels = torch.tensor([1, 2, 1][:B]) if O == 2 else torch.ones(B, dtype=torch.long)
    case = synth.make_feature_case(B=B, O=O, T=T, seed=seed, labels=labels)
    g = torch.Generator().manual_seed(seed)
    src0, src1 = min(T - 1, 7), 2
    groups = []                              # per object: [(source template, [ids holding a copy of it])]
    for o in range(O):
        b = int((case.q_label == o + 1).nonzero()[0, 0])
        case.bank_feat[o, src0] = case.q_feat[b]
        case.bank_feat[o, src1] = torch.nn.functional.normalize(case.q_feat[b] + 0.03 * torch.randn(P, 1024, generator=g),
                                                                dim=-1)
        case.bank_mask16[o, [src0, src1]] = case.q_mask16[b]
        g0 = [i for i in G0 if i < T and i not in (src0, src1)]
        g1 = [i for i in G1 if i < T and i not in (src0, src1)]
        for src, ids in ((src0, g0), (src1, g1)):
            case.bank_feat[o, ids] = case.bank_feat[o, src].clone()
            case.bank_mask16[o, ids] = case.bank_mask16[o, src].clone()
        groups.append([(src0, g0), (src1, g1)])
    if B == 3:
        case.q_mask16[2] = 0                 # fully masked query: every score is 0
    return case, groups


def _expected_topk(sim_avg, groups, k):
    """Winners by (score desc, id asc) over the oracle's scores, with each planted copy given its source's score; checks
    that every decision near the top-k is either a planted tie, a tie at exactly 0, or at least GAP apart."""
    sim = sim_avg.double().clone()
    gid = list(range(len(sim)))
    for src, ids in groups:
        sim[ids] = float(sim[src])
        for i in ids:
            gid[i] = src
    vals = sim.tolist()
    order = python_topk(vals, list(range(len(vals))), len(vals))
    head = order[:k + 1]
    for a, b in zip(head, head[1:]):
        if vals[a] == vals[b]:
            assert gid[a] == gid[b] or vals[a] == 0.0, f"unplanted oracle tie between templates {a} and {b}"
        else:
            assert vals[a] - vals[b] > GAP, f"templates {a} / {b} only {vals[a] - vals[b]:.2e} apart in the oracle"
    return order[:k], vals


@pytest.mark.parametrize("T,k,B", TOPK_CASES)
def test_topk_select_picks_the_python_sort_with_planted_ties(T, k, B):
    """sim_topk / sim_candidates against a Python sort of the oracle's per-template scores, by (score descending,
    template id ascending).  Identical templates are planted at ids in one thread (256 apart), in other lanes and in
    other warps: their scores are bit-identical, and the lower id must win, in order.  The winners' records (score_pts,
    src_pts, tar_pts) are those of the oracle's template.  A fully masked query scores 0 everywhere: ids 0..k-1."""
    case, groups = _planted_topk_case(T, B, seed=3 * T + k)
    eng = engine_from_case(case, k=k)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    cand = eng.alloc_candidates(B)
    cand["score"].fill_(float("nan"))
    cand["id"].fill_(SENT)
    cand["pts_score"].fill_(float("nan"))
    cand["idx"].fill_(0xAB)
    cand["valid"].fill_(0xAB)
    eng.sim_candidates(cand)
    m = sentinel_matches(B, k)
    check(_lib_().gp_sim_topk(eng._h, B, C.byref(_matches_struct(m)), _stream()))
    torch.cuda.synchronize(DEV)
    m = {kk: v.cpu() for kk, v in m.items()}
    ri = synth.to_reference_layout(case)
    ref = port.similarity_search(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"], k=k,
                                 return_intermediates=True)
    ties_seen, pts_err, src_err = 0, 0.0, 0.0
    for b in range(B):
        o = int(case.q_label[b]) - 1
        want, vals = _expected_topk(ref["sim_avg"][b], groups[o], k)
        got = m["id_src"][b].tolist()
        assert got == want, f"query {b}: kernel {got}, Python sort {want}"
        src_err = max(src_err, float((m["score_src"][b].double() - torch.tensor([vals[i] for i in want])).abs().max()))
        for src, ids in groups[o]:
            pos = [j for j, i in enumerate(got) if i == src or i in ids]
            if len(pos) > 1:
                ties_seen += 1
                tied = bits(m["score_src"][b, pos])
                assert bool((tied == tied[0]).all()), f"query {b}: planted copies of {src} scored differently"
        sel = torch.tensor(want)
        valid = ref["mask_all"][b, sel] != 0
        assert torch.equal(m["src_pts"][b], pts_of(valid, ref["idx_tar2src"][b, sel]))
        assert torch.equal(m["tar_pts"][b], pts_of(valid, torch.arange(P).expand(k, P)))
        pts_err = max(pts_err, float((m["score_pts"][b] - ref["score_tar2src"][b, sel]).abs().max()))
        if B == 3 and b == 2:
            assert got == list(range(k)) and bool((m["score_src"][b] == 0).all())
    write_report(f"tail_topk_select_T{T}_k{k}.json", {"score_pts": pts_err, "score_src": src_err})
    assert pts_err < BAR_SCORE_PTS and src_err < BAR_SCORE_PTS, f"score_pts {pts_err:.3e}, score_src {src_err:.3e}"
    if k > 1:
        assert ties_seen > 0, "no planted tie reached the top-k"
    # the candidate records of sim_candidates are the same winners (single GPU: global id = local id)
    assert torch.equal(cand["id"].cpu()[0].long(), m["id_src"])
    assert torch.equal(bits(cand["score"].cpu()[0]), bits(m["score_src"]))
    assert torch.equal(bits(cand["pts_score"].cpu()[0]), bits(m["score_pts"]))
    assert bool((cand["valid"].cpu()[0] <= 1).all())


def test_topk_select_orders_negative_scores_at_a_threshold_below_0():
    """sim_threshold = -0.5 keeps negative similarities.  Eight templates anti-aligned with the query (every similarity
    about -0.19, full masks) get negative per-template scores, which must rank below the positive and zero scores in
    the same (score, id) order as the oracle."""
    T, k = 24, 20
    case = synth.make_feature_case(B=1, O=1, T=T, seed=31)
    g = torch.Generator().manual_seed(33)
    unit = lambda x: torch.nn.functional.normalize(x, dim=-1)
    c = unit(torch.randn(1024, generator=g))
    case.q_mask16[0] = 1                     # a masked query patch would add a 0 to every column, beating the negatives
    case.q_feat[0] = unit(c + 0.3 * unit(torch.randn(P, 1024, generator=g)))
    neg, pos = [1, 4, 8, 11, 13, 17, 20, 23], [2, 6, 15]
    for n, sgn in [(n, -1.0) for n in neg] + [(n, 1.0) for n in pos]:
        case.bank_feat[0, n] = unit(sgn * 0.2 * c + unit(torch.randn(P, 1024, generator=g)))
        case.bank_mask16[0, n] = 1
    eng = engine_from_case(case, k=k, sim_threshold=-0.5)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    m = sentinel_matches(1, k)
    check(_lib_().gp_sim_topk(eng._h, 1, C.byref(_matches_struct(m)), _stream()))
    torch.cuda.synchronize(DEV)
    ri = synth.to_reference_layout(case)
    ref = port.similarity_search(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"], k=k,
                                 sim_threshold=-0.5, return_intermediates=True)
    want, vals = _expected_topk(ref["sim_avg"][0], [], k)
    assert sum(v < 0 for v in vals) >= 3 and min(vals[i] for i in want) < 0, "no negative score in the top-k"
    assert m["id_src"][0].tolist() == want
    assert torch.allclose(m["score_src"][0].cpu().double(), torch.tensor([vals[i] for i in want], dtype=torch.float64),
                          atol=2e-6, rtol=0)


def test_topk_select_pads_a_shard_with_fewer_than_k_templates():
    """A shard holding 2 of 5 templates (rank 1 of 3: global ids 1 and 4) at k = 5 emits its two templates by score,
    then three padding records: score -inf, id 0x7fffffff, pts_score 0, idx 0, valid 0."""
    case = synth.make_feature_case(B=2, O=1, T=5, seed=41)
    eng = engine_from_case(case, k=5, shard_rank=1, shard_world=3)
    eng.set_queries(case.q_feat, case.q_mask16.reshape(-1, 16, 16), case.q_label - 1)
    cand = eng.alloc_candidates(2)
    cand["score"].fill_(float("nan"))
    cand["id"].fill_(SENT)
    cand["pts_score"].fill_(float("nan"))
    cand["idx"].fill_(0xAB)
    cand["valid"].fill_(0xAB)
    eng.sim_candidates(cand)
    torch.cuda.synchronize(DEV)
    c = {kk: v.cpu()[0] for kk, v in cand.items()}
    ri = synth.to_reference_layout(case)
    ref = port.similarity_search(ri["src_feats"], ri["tar_feat"], ri["src_masks"], ri["tar_mask"], k=5,
                                 return_intermediates=True)
    for b in range(2):
        s = ref["sim_avg"][b]
        want = sorted([1, 4], key=lambda i: (-float(s[i]), i))
        assert abs(float(s[1]) - float(s[4])) > GAP
        assert c["id"][b, :2].tolist() == want
        assert torch.allclose(c["score"][b, :2], s[want], atol=2e-6, rtol=0)
        assert bool((c["score"][b, 2:] == -math.inf).all()) and c["id"][b, 2:].tolist() == [PAD_ID] * 3
        assert bool((c["pts_score"][b, 2:] == 0).all()) and not bool(c["idx"][b, 2:].any())
        assert not bool(c["valid"][b, 2:].any())
        valid = ref["mask_all"][b, want] != 0
        assert torch.equal(c["valid"][b, :2].bool(), valid)
        assert torch.equal(c["idx"][b, :2].long()[valid], ref["idx_tar2src"][b, want][valid])


# ========================================================================================================= top-k merge
MERGE_CASES = [(1, 5), (2, 5), (3, 5), (12, 5), (8, 8), (2, 32)]     # G * k up to the 64-bit `used` mask


def _merge_inputs(G, B, k, seed):
    """G per-shard candidate lists as topk_select_kernel writes them: global id = local * G + g, each list sorted by
    (score desc, id asc), quantised scores (exact ties inside and across shards, some negative), the last shard of a
    multi-shard case holding fewer than k templates (padding records)."""
    rng = np.random.default_rng(seed)
    score = np.zeros((G, B, k), np.float32)
    ids = np.zeros((G, B, k), np.int32)
    valid = (rng.random((G, B, k, P)) < 0.7).astype(np.uint8)
    idx = rng.integers(0, 256, (G, B, k, P)).astype(np.uint8)
    pts = rng.standard_normal((G, B, k, P)).astype(np.float32)
    for g in range(G):
        n_real = k // 2 + 1 if (G > 1 and g == G - 1) else k
        for b in range(B):
            local = rng.choice(max(3 * k, 40), n_real, replace=False)
            s = (rng.integers(0, 6, n_real) / 8 - 0.125).astype(np.float32)
            gid = (local * G + g).astype(np.int32)
            order = sorted(range(n_real), key=lambda i: (-s[i], gid[i]))
            score[g, b, :n_real], ids[g, b, :n_real] = s[order], gid[order]
            score[g, b, n_real:], ids[g, b, n_real:] = -np.inf, PAD_ID
            valid[g, b, n_real:], idx[g, b, n_real:], pts[g, b, n_real:] = 0, 0, 0
    rel_scale = rng.standard_normal((G, B, k, P)).astype(np.float32)
    rel_inplane = rng.standard_normal((G, B, k, P, 2)).astype(np.float32)
    return dict(score=score, id=ids, pts_score=pts, idx=idx, valid=valid, rel_scale=rel_scale, rel_inplane=rel_inplane)


FIELDS = ("score", "id", "pts_score", "idx", "valid", "rel_scale", "rel_inplane")


@pytest.mark.parametrize("packed", [False, True], ids=["dense", "packed"])
@pytest.mark.parametrize("G,k", MERGE_CASES)
def test_topk_merge_against_python_sort(G, k, packed):
    """Engine.topk_merge's kernel on caller-made candidate lists, dense ([G][B][k] per field) or packed (one record
    per rank, rank_stride_bytes apart): id_src / score_src / score_pts are the winners' in (score desc, global id asc)
    order, tar_pts / src_pts are their expansion from valid / idx, and rel_scale / rel_inplane are copied bit for bit."""
    B = 3
    eng = Engine(1, k, B, device=DEV, k=k)
    eng.set_queries(torch.zeros(B, P, 1024), torch.ones(B, 16, 16), torch.zeros(B, dtype=torch.int32), norm_passes=0)
    h = _merge_inputs(G, B, k, seed=10 * G + k)
    keep = []
    if packed:
        sizes = [h[f][0].nbytes for f in FIELDS]
        offs = np.cumsum([0] + [(s + 255) // 256 * 256 for s in sizes])
        stride = int(offs[-1])
        buf = torch.zeros(G, stride, dtype=torch.uint8)
        for f, o, s in zip(FIELDS, offs, sizes):
            buf[:, o:o + s] = torch.from_numpy(h[f].reshape(G, -1).view(np.uint8).copy())
        buf = buf.to(DEV)
        keep.append(buf)
        ptrs = [buf.data_ptr() + int(o) for o in offs[:-1]]
    else:
        stride = 0
        dev = [torch.from_numpy(h[f]).to(DEV) for f in FIELDS]
        keep += dev
        ptrs = [t.data_ptr() for t in dev]
    cs = _lib.GpCandidates(*ptrs)
    m = sentinel_matches(B, k)
    rs, ri = nan_f32(B, k, P), nan_f32(B, k, P, 2)
    check(_lib_().gp_topk_merge(eng._h, B, G, C.byref(cs), stride, C.byref(_matches_struct(m)), rs.data_ptr(),
                                ri.data_ptr(), _stream()))
    torch.cuda.synchronize(DEV)
    m = {kk: v.cpu() for kk, v in m.items()}
    t = {f: torch.from_numpy(h[f]) for f in FIELDS}
    for b in range(B):
        cands = python_topk(h["score"][:, b].reshape(-1).tolist(), h["id"][:, b].reshape(-1).tolist(), k)
        g = torch.tensor([c // k for c in cands])
        j = torch.tensor([c % k for c in cands])
        assert m["id_src"][b].tolist() == t["id"][g, b, j].tolist(), f"query {b}"
        assert torch.equal(bits(m["score_src"][b]), bits(t["score"][g, b, j]))
        assert torch.equal(bits(m["score_pts"][b]), bits(t["pts_score"][g, b, j]))
        v = t["valid"][g, b, j] != 0
        assert torch.equal(m["tar_pts"][b], pts_of(v, torch.arange(P).expand(k, P)))
        assert torch.equal(m["src_pts"][b], pts_of(v, t["idx"][g, b, j].long()))
        assert torch.equal(bits(rs.cpu()[b]), bits(t["rel_scale"][g, b, j]))
        assert torch.equal(bits(ri.cpu()[b]), bits(t["rel_inplane"][g, b, j]))


# ======================================================================================================== IST regressor
def _ist_engine(form, monkeypatch, rank, world, ist_global, O=2, Tg=12, max_batch=4, k=5):
    monkeypatch.setenv("GIGAPOSE_MLP_SIMT", "1" if form == "simt" else "0")
    local = list(range(rank, Tg, world))
    eng = Engine(O, len(local), max_batch, device=DEV, k=k, shard_rank=rank, shard_world=world,
                 num_templates_global=Tg, ist_bank_global=ist_global)
    g = torch.Generator().manual_seed(51)
    bank_ist = torch.randn(O, Tg, 256, 16, 16, generator=g)
    for o in range(O):
        eng.bank_write(o, 0, torch.zeros(len(local), P, 1024), torch.ones(len(local), 16, 16), norm_passes=0)
        eng.bank_write_ist(o, 0, bank_ist[o] if ist_global else bank_ist[o, local])
    reg = port.RegressorPort(seed=52)
    eng.set_ist_weights(reg)
    q_obj = torch.tensor([1, 0, 1, 1][:max_batch], dtype=torch.int32)
    eng.set_queries(torch.zeros(max_batch, P, 1024), torch.ones(max_batch, 16, 16), q_obj, norm_passes=0)
    return eng, reg, bank_ist, q_obj, local


def _ist_matches(B, k, local, world, rank, pattern, seed):
    """id_src from this shard's templates; `pattern`: 'random' (per-row valid fractions from 0 to 1, row (0,0) with
    nothing valid and row (0,1) all valid), 'none' or 'all'."""
    g = torch.Generator().manual_seed(seed)
    lid = torch.tensor(local)[torch.randint(0, len(local), (B, k), generator=g)]
    assert bool(((lid - rank) % world == 0).all())
    src = torch.randint(0, 16, (B, k, P, 2), generator=g)
    tar = torch.randint(0, 16, (B, k, P, 2), generator=g)
    if pattern == "random":
        frac = torch.rand(B, k, 1, generator=g)
        frac[0, 0], frac[0, 1] = 0.0, 1.01
        valid = torch.rand(B, k, P, generator=g) < frac
    else:
        valid = torch.full((B, k, P), pattern == "all")
    src[~valid] = -1
    tar[~valid] = -1
    z = torch.zeros(B, k, P)
    return dict(id_src=lid, score_src=z[..., 0].clone(), score_pts=z, tar_pts=tar, src_pts=src), valid


def run_ist(eng, q_ist, m, b0):
    n = q_ist.shape[0]
    md = {kk: v.to(DEV).contiguous() for kk, v in m.items()}
    rs, ri = nan_f32(n, eng.k, P), nan_f32(n, eng.k, P, 2)
    q = q_ist.to(DEV).contiguous()
    check(_lib_().gp_ist_mlp(eng._h, b0, n, q.data_ptr(), _lib.LAYOUT_CHANNEL_MAJOR, C.byref(_matches_struct(md)),
                             rs.data_ptr(), ri.data_ptr(), _stream()))
    torch.cuda.synchronize(DEV)
    return rs.cpu(), ri.cpu()


def mlp64(reg, rows):
    """fp64 forward of both heads, and each output's propagated magnitude |W3| (|W2| (|W1||x| + |b1|) + |b2|) + |b3|."""
    out = []
    for head in (reg.scale_predictor, reg.inplane_predictor):
        x, den = rows, rows.abs()
        for i in (0, 2, 4):
            W, b = head[i].weight.detach().double(), head[i].bias.detach().double()
            x, den = x @ W.T + b, den @ W.abs().T + b.abs()
            if i < 4:
                x = x.clamp(min=0)
        if isinstance(head[-1], torch.nn.Tanh):
            x = torch.tanh(x)
        out.append((x, den))
    return out


def ist_reference(reg, q_ist, bank_ist, q_obj, m, valid):
    b, kk, t = valid.nonzero(as_tuple=True)
    tar, src = m["tar_pts"][b, kk, t], m["src_pts"][b, kk, t]
    qf = q_ist[b, :, tar[:, 1], tar[:, 0]]
    tf = bank_ist[q_obj.long()[b], m["id_src"][b, kk], :, src[:, 1], src[:, 0]]
    return mlp64(reg, torch.cat([qf, tf], 1).double())


@pytest.mark.parametrize("layout", ["single", "shard", "ist_global"])
@pytest.mark.parametrize("form", ["simt", "tc"])
def test_ist_regressor_against_fp64(form, layout, monkeypatch):
    """gp_ist_mlp on caller-made matches, in the fp32 SIMT form and the fp16-pair tensor-core form: the outputs of the
    valid slots against an fp64 forward of the same weights on the gathered rows, normalised by the propagated
    magnitude; every invalid slot holds exactly -1000.  Rows are compacted through an atomicAdd, so their order varies:
    two calls, and the windows [1, 3) and [3, 4) of the batch, must give the same bits.  The templates are gathered
    through the shard map ((id - 1) / 3 on rank 1 of 3) or by global id (ist_bank_global).  Row counts: 0, all
    4 x 5 x 256 slots, and a random pattern whose count is not a multiple of 64."""
    rank, world = (0, 1) if layout == "single" else (1, 3)
    eng, reg, bank_ist, q_obj, local = _ist_engine(form, monkeypatch, rank, world, layout == "ist_global")
    B, k = 4, eng.k
    q_ist = torch.randn(B, 256, 16, 16, generator=torch.Generator().manual_seed(53))
    report = {}
    for pattern in ("random", "none", "all"):
        m, valid = _ist_matches(B, k, local, world, rank, pattern, seed=54)
        nvalid = int(valid.sum())
        if pattern == "random":
            assert nvalid % 64 != 0 and not bool(valid[0, 0].any()) and bool(valid[0, 1].all())
        rs, ri = run_ist(eng, q_ist, m, 0)
        assert bool((rs[~valid] == -1000.0).all()) and bool((ri[~valid] == -1000.0).all()), "invalid slot not -1000"
        rs2, ri2 = run_ist(eng, q_ist, m, 0)
        assert torch.equal(bits(rs), bits(rs2)) and torch.equal(bits(ri), bits(ri2)), "two calls differ"
        for b0, n in ((1, 2), (3, 1)):
            w = {kk: v[b0:b0 + n] for kk, v in m.items()}
            rsw, riw = run_ist(eng, q_ist[b0:b0 + n], w, b0)
            assert torch.equal(bits(rsw), bits(rs[b0:b0 + n])) and torch.equal(bits(riw), bits(ri[b0:b0 + n])), \
                f"window [{b0}, {b0 + n}) differs from the whole batch"
        if nvalid == 0:
            continue
        (s64, sden), (i64, iden) = ist_reference(reg, q_ist, bank_ist, q_obj, m, valid)
        es = float(((rs[valid].double() - s64[:, 0]).abs() / sden[:, 0]).max())
        ei = float(((ri[valid].double() - i64).abs() / iden).max())
        report[pattern] = {"rows": nvalid, "scale": es, "inplane": ei}
        assert max(es, ei) < BAR_MLP[form], f"{pattern}: scale {es:.3e}, in-plane {ei:.3e}"
    write_report(f"tail_ist_{form}_{layout}.json", report)


# ============================================================================================================== RANSAC
def ransac_f32(src_pts, tar_pts, rel_scale, rel_inplane, thr, patch_size):
    """ransac_kernel restated in numpy float32, vectorised over the n x n (candidate, correspondence) pairs, in the
    kernel's operation order: every product and sum rounded to fp32, no fused multiply-add, the proposer transform's
    `+ 0.0f`, the first maximum.  Also returns each pair's decision matrix for the fp64 comparison."""
    f = np.float32
    N = src_pts.shape[0]
    M = np.zeros((N, 3, 3), f)
    failed = np.zeros(N, np.uint8)
    count = np.zeros(N, np.int32)
    in_src = np.full((N, P, 2), -1, np.int64)
    in_tar = np.full((N, P, 2), -1, np.int64)
    in_sc = np.zeros((N, P), np.int64)
    thr, ps = f(thr), f(patch_size)
    detail = []
    for i in range(N):
        keep = np.nonzero(src_pts[i, :, 0] != -1)[0]
        n = len(keep)
        if n == 0:
            M[i] = np.eye(3, dtype=f)
            detail.append(None)
            continue
        si, ti = src_pts[i, keep], tar_pts[i, keep]
        sx, sy = si[:, 0].astype(f) * ps, si[:, 1].astype(f) * ps
        tx, ty = ti[:, 0].astype(f) * ps, ti[:, 1].astype(f) * ps
        sc = rel_scale[i, keep]
        c, s = rel_inplane[i, keep, 0], rel_inplane[i, keep, 1]
        m00, m01, m10, m11 = c * sc, (-s) * sc, s * sc, c * sc
        ax = (m00 * sx + m01 * sy) + f(0.0)
        ay = (m10 * sx + m11 * sy) + f(0.0)
        m02, m12 = tx - ax, ty - ay
        px = (m00[:, None] * sx[None, :] + m01[:, None] * sy[None, :]) + m02[:, None]
        py = (m10[:, None] * sx[None, :] + m11[:, None] * sy[None, :]) + m12[:, None]
        dx, dy = tx[None, :] - px, ty[None, :] - py
        err = np.sqrt(dx * dx + dy * dy)
        inl = err <= thr
        np.fill_diagonal(inl, False)
        score = inl.sum(1)
        best = int(np.argmax(score))
        failed[i] = score[best] == 0
        count[i] = score[best]
        M[i] = [[m00[best], m01[best], m02[best]], [m10[best], m11[best], m12[best]], [0, 0, 1]]
        j = np.nonzero(inl[best])[0]
        in_src[i, :len(j)], in_tar[i, :len(j)], in_sc[i, :len(j)] = si[j], ti[j], 1
        detail.append((keep, inl))
    return dict(M=M, failed=failed, count=count, in_src=in_src, in_tar=in_tar, in_sc=in_sc), detail


def ransac_f64_decisions(src_pts, tar_pts, rel_scale, rel_inplane, thr, patch_size, i, keep):
    """fp64 inlier decisions of pair i over its n x n candidates, and the margin within which fp32 may decide otherwise:
    2^-18 of the magnitudes summed into each coordinate."""
    si, ti = src_pts[i, keep].astype(np.float64) * patch_size, tar_pts[i, keep].astype(np.float64) * patch_size
    sc = rel_scale[i, keep].astype(np.float64)
    c, s = rel_inplane[i, keep, 0].astype(np.float64), rel_inplane[i, keep, 1].astype(np.float64)
    m00, m01, m10, m11 = c * sc, -s * sc, s * sc, c * sc
    m02 = ti[:, 0] - (m00 * si[:, 0] + m01 * si[:, 1])
    m12 = ti[:, 1] - (m10 * si[:, 0] + m11 * si[:, 1])
    ux, uy = m00[:, None] * si[None, :, 0], m01[:, None] * si[None, :, 1]
    vx, vy = m10[:, None] * si[None, :, 0], m11[:, None] * si[None, :, 1]
    dx = ti[None, :, 0] - (ux + uy + m02[:, None])
    dy = ti[None, :, 1] - (vx + vy + m12[:, None])
    err = np.sqrt(dx * dx + dy * dy)
    mag = np.maximum(np.abs(ux) + np.abs(uy) + np.abs(m02)[:, None] + np.abs(ti[None, :, 0]),
                     np.abs(vx) + np.abs(vy) + np.abs(m12)[:, None] + np.abs(ti[None, :, 1]))
    return err <= thr, np.abs(err - thr) <= 2.0 ** -18 * mag


TIE_PAIR = 14                                                           # index of the cross-warp tie in _ransac_inputs
LATTICE = [(2 * a, 2 * b) for a in range(-3, 4) for b in range(-3, 4)]   # offsets >= 2 patches apart


def _with_offset(rng, d):
    """(src, tar) patch pair with tar - src = d, both inside the 16 x 16 grid."""
    sx = rng.integers(max(0, -d[0]), min(16, 16 - d[0]))
    sy = rng.integers(max(0, -d[1]), min(16, 16 - d[1]))
    return (sx, sy), (sx + d[0], sy + d[1])


def _ransac_inputs(seed):
    """About 1 000 (detection, hypothesis) pairs [N, 256]: invalid slots hold -1 points and the regressor's -1000."""
    rng = np.random.default_rng(seed)
    pairs = []

    def new():
        p = dict(src=np.full((P, 2), -1, np.int64), tar=np.full((P, 2), -1, np.int64),
                 sc=np.full(P, -1000, np.float32), cs=np.full((P, 2), -1000, np.float32))
        pairs.append(p)
        return p

    def put(p, t, src, tar, sc=1.0, c=1.0, s=0.0):
        p["src"][t], p["tar"][t], p["sc"][t], p["cs"][t] = src, tar, sc, (c, s)

    for _ in range(3):                                   # n = 0: identity, not failed
        new()
    for t in (0, 117, 255):                              # n = 1: failed
        put(new(), t, (3, 4), (5, 6), 1.3, 0.8, 0.6)
    p = new()                                            # n = 2, each the other's inlier
    put(p, 10, (2, 2), (4, 5))
    put(p, 200, (9, 1), (11, 4))
    for invalid in ((0,), (255,), (0, 255), ()):         # n = 255 / 254 / 256 with invalid slots at the ends
        p = new()
        for t in range(P):
            if t not in invalid:
                src, tar = _with_offset(rng, LATTICE[rng.integers(0, 6)])
                put(p, t, src, tar, 1.0 + 0.01 * rng.standard_normal(), 1.0, 0.0)
    for n in (40, 100, 256):                             # whole-patch offsets at scale 1, rotation 0: err = k * patch
        p = new()                                        # exactly (e.g. 14 on the threshold), diagonals at k * 14 sqrt 2
        slots = rng.choice(P, n, replace=False)
        for t in slots:
            d = [(0, 0), (1, 0), (0, 1), (-1, 0), (1, 1), (2, 0), (0, -2)][rng.integers(0, 7)]
            put(p, t, *_with_offset(rng, d))
    assert len(pairs) == TIE_PAIR
    p = new()                                            # equal best scores in warps 1 and 6: the first (slot 32) wins
    others = [d for d in LATTICE if d not in ((0, 0), (6, 6))]
    for t in range(P):
        d = (0, 0) if 32 <= t < 52 else (6, 6) if 192 <= t < 212 else others[t % len(others)]
        put(p, t, *_with_offset(rng, d))
    p = new()                                            # 30 isolated correspondences: every score 0, failed
    for j, t in enumerate(rng.choice(P, 30, replace=False)):
        put(p, t, *_with_offset(rng, LATTICE[j]))
    for _ in range(6):                                   # one consistent model with regressor noise: organic knife edges
        p = new()
        a = rng.uniform(-0.3, 0.3)
        for t in rng.choice(P, rng.integers(20, 257), replace=False):
            src, tar = _with_offset(rng, (int(rng.integers(-2, 3)), int(rng.integers(-2, 3))))
            put(p, t, src, tar, 1 + 0.05 * rng.standard_normal(), math.cos(a) + 0.03 * rng.standard_normal(),
                math.sin(a) + 0.03 * rng.standard_normal())
    while len(pairs) < 1000:                             # random-weight regressor magnitudes: scales to +-100,
        p = new()                                        # translations ~1e4 px; correspondences share source patches
        n = int(rng.choice([2, 5, 17, 64, 128, 200, 256]))
        srcs = rng.integers(0, 16, (4, 2))
        for t in rng.choice(P, n, replace=False):
            put(p, t, srcs[rng.integers(0, 4)], rng.integers(0, 16, 2), rng.uniform(-100, 100), rng.uniform(-1, 1),
                rng.uniform(-1, 1))
    st = lambda key: np.stack([q[key] for q in pairs])
    return st("src"), st("tar"), st("sc"), st("cs")


@pytest.mark.parametrize("patch_size", [14, 8])
@pytest.mark.parametrize("thr", [14.0, 7.5, 0.0])
def test_ransac_is_bit_exact_to_the_float32_restatement(thr, patch_size):
    """gp_ransac on 1 000 pairs equals `ransac_f32` bit for bit: M, failed, inlier_count, the compacted inlier points
    and scores and their -1 / -1 / 0 tails.  Covered: n = 0 (identity, not failed), 1 (failed), 2, 254-256 with invalid
    slots at t = 0 / 255, distances of exactly the threshold (whole-patch offsets at scale 1), equal best scores in
    different warps, all scores 0, and scales to +-100.  Every fp32 inlier decision equals the fp64 decision unless the
    fp64 distance lies within 2^-18 of the coordinates' magnitudes from the threshold; those are counted."""
    src, tar, sc, cs = _ransac_inputs(seed=60)
    N = src.shape[0]
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    out = dict(M=nan_f32(N, 3, 3), failed=torch.full((N,), 0xAB, dtype=torch.uint8, device=DEV),
               in_src=sent_i64(N, P, 2), in_tar=sent_i64(N, P, 2), in_sc=sent_i64(N, P),
               count=torch.full((N,), SENT, dtype=torch.int32, device=DEV))
    ro = _lib.GpRansacOut(*(out[kk].data_ptr() for kk in ("M", "failed", "in_src", "in_tar", "in_sc", "count")))
    ins = [d(src), d(tar), d(sc), d(cs)]
    check(_lib_().gp_ransac(N, C.c_float(thr), patch_size, *(t.data_ptr() for t in ins), C.byref(ro), _stream()))
    torch.cuda.synchronize(DEV)
    got = {kk: v.cpu().numpy() for kk, v in out.items()}
    want, detail = ransac_f32(src, tar, sc, cs, thr, patch_size)
    assert np.array_equal(got["M"].view(np.int32), want["M"].view(np.int32)), \
        f"M differs in {int((got['M'] != want['M']).any(axis=(1, 2)).sum())} pairs"
    for kk in ("failed", "count", "in_src", "in_tar", "in_sc"):
        assert np.array_equal(got[kk], want[kk]), f"{kk} differs in {int((got[kk] != want[kk]).reshape(N, -1).any(1).sum())} pairs"
    decisions = near = 0
    for i, dt in enumerate(detail):
        if dt is None:
            continue
        keep, inl = dt
        d64, margin = ransac_f64_decisions(src, tar, sc, cs, thr, patch_size, i, keep)
        np.fill_diagonal(d64, False)
        np.fill_diagonal(margin, False)
        off = ~np.eye(len(keep), dtype=bool)
        bad = (inl != d64) & ~margin & off
        assert not bad.any(), f"pair {i}: {int(bad.sum())} decisions differ from fp64 outside the margin"
        decisions += int(off.sum())
        near += int((margin & off).sum())
    # the planted cases are live
    assert want["count"][:3].tolist() == [0, 0, 0] and not want["failed"][:3].any()
    assert want["failed"][3:6].all() and want["count"][6] == 1
    assert want["count"][TIE_PAIR] == 19 and want["M"][TIE_PAIR, :2, 2].tolist() == [0.0, 0.0]
    assert want["failed"][TIE_PAIR + 1] and want["count"][TIE_PAIR + 1] == 0
    write_report(f"tail_ransac_thr{thr}_ps{patch_size}.json",
                 {"pairs": N, "decisions": decisions, "within_margin": near,
                  "inliers": int(want["count"].sum()), "failed": int(want["failed"].sum())})


# ======================================================================================================= sort and pose
def _rotations(n, rng):
    q, r = np.linalg.qr(rng.standard_normal((n, 3, 3)))
    q = q * np.sign(np.diagonal(r, axis1=1, axis2=2))[:, None, :]
    q[np.linalg.det(q) < 0, :, 0] *= -1
    return q


def _crop_M(n, rng):
    s = rng.uniform(0.3, 3.0, n)
    M = np.zeros((n, 3, 3))
    M[:, 0, 0] = M[:, 1, 1] = s
    M[:, 0, 2] = 112 - s * rng.uniform(150, 490, n)
    M[:, 1, 2] = 112 - s * rng.uniform(120, 360, n)
    M[:, 2, 2] = 1
    return M


def _similarity(angle, scale, t):
    c, s = math.cos(angle), math.sin(angle)
    return np.array([[scale * c, -scale * s, t[0]], [scale * s, scale * c, t[1]], [0, 0, 1]])


def _pose_inputs(O, T, B, k, seed):
    """Template poses with proper random rotations and tz in [300, 1500] mm, crop matrices with scales 0.3 .. 3, a
    query K with non-zero off-diagonal terms, and RANSAC similarities at 0, 90 and 180 degrees, random angles, and the
    identity of n = 0."""
    rng = np.random.default_rng(seed)
    tK = np.tile(np.array(synth.LM_K), (O, 1, 1))
    tM = _crop_M(O * T, rng).reshape(O, T, 3, 3)
    tP = np.zeros((O, T, 4, 4))
    tP[..., :3, :3] = _rotations(O * T, rng).reshape(O, T, 3, 3)
    tP[..., 0, 3], tP[..., 1, 3] = rng.uniform(-100, 100, (O, T)), rng.uniform(-100, 100, (O, T))
    tP[..., 2, 3] = rng.uniform(300, 1500, (O, T))
    tP[..., 3, 3] = 1
    qK = np.tile(np.array(synth.LM_K), (B, 1, 1))
    qK[:, 0, 1], qK[:, 1, 0] = rng.uniform(-3, 3, B), rng.uniform(-2, 2, B)
    qK[:, 2, 0], qK[:, 2, 1] = rng.uniform(-1e-4, 1e-4, B), rng.uniform(-1e-4, 1e-4, B)
    qM = _crop_M(B, rng)
    M = np.zeros((B, k, 3, 3))
    for b in range(B):
        for j in range(k):
            kind = j % 5
            if kind == 0:
                M[b, j] = np.eye(3)
            else:
                ang = [0.0, math.pi / 2, math.pi, rng.uniform(-math.pi, math.pi)][kind - 1]
                M[b, j] = _similarity(ang, rng.uniform(0.5, 2.0), rng.uniform(-60, 60, 2))
    f = lambda a: torch.from_numpy(a).float()
    return dict(tK=f(tK), tM=f(tM), tP=f(tP), qK=f(qK), qM=f(qM), M=f(M))


def pose64(q_obj, qK, qM, id_src, M, tK, tM, tP):
    """port.pose_recovery in fp64 on the fp32 inputs (object index given 0-based)."""
    d = lambda t: t.double()
    qK, qM, M, tK, tM, tP = map(d, (qK, qM, M, tK, tM, tP))
    B, k = id_src.shape
    o = q_obj.long()[:, None].expand(B, k)
    tKb, tMb, P_ = tK[o], tM[o, id_src], tP[o, id_src].clone()
    sc = M[..., :2, 0].norm(dim=-1)
    Rin = torch.eye(3, dtype=torch.float64).repeat(B, k, 1, 1)
    Rin[..., :2, :2] = M[..., :2, :2] / sc[..., None, None]
    R = Rin @ P_[..., :3, :3]
    tz = P_[..., 2, 3]
    c2d = tKb @ P_[..., :3, 3:4]
    c2d = c2d / c2d[..., 2:3, :]
    qs = qM[:, 0, 0]
    Minv = torch.eye(3, dtype=torch.float64).repeat(B, 1, 1)
    Minv[:, 0, 0] = Minv[:, 1, 1] = 1 / qs
    Minv[:, :2, 2] = -qM[:, :2, 2] / qs[:, None]
    aff = Minv[:, None] @ M @ tMb
    qc = aff @ c2d
    s2d = aff[..., :2, 0].norm(dim=-1)
    qz = (tz / s2d) * (qK[:, None, 0, 0] / tKb[..., 0, 0])
    tr = (torch.inverse(qK)[:, None] @ qc)[..., 0]
    tr = tr / tr[..., 2:3] * qz[..., None]
    out = P_
    out[..., :3, :3] = R
    out[..., :3, 3] = tr
    return out


def pose_err(got, ref):
    e = (got.double() - ref).abs()
    et = e[..., :3, 3] / ref[..., :3, 3].abs().clamp(min=1.0)
    return float(e[..., :3, :3].max()), float(et.max()), bool(torch.equal(got[..., 3, :].double(), ref[..., 3, :]))


def _pose_engine(O, T, B, k, q_obj, inp):
    eng = Engine(O, T, B, device=DEV, k=k)
    eng.set_poses(inp["tK"], inp["tM"], inp["tP"])
    eng.set_queries(torch.zeros(B, P, 1024), torch.ones(B, 16, 16), q_obj, norm_passes=0)
    return eng


def run_sort_and_pose(eng, b0, n, sort, qK, qM, m, rel_scale, rel_inplane, r):
    k = eng.k
    o = sentinel_matches(n, k)
    o.update(relScale=nan_f32(n, k, P), relInplane=nan_f32(n, k, P, 2), M=nan_f32(n, k, 3, 3),
             failed=torch.full((n, k), 0xAB, dtype=torch.uint8, device=DEV), in_src=sent_i64(n, k, P, 2),
             in_tar=sent_i64(n, k, P, 2), in_sc=sent_i64(n, k, P), scores=nan_f32(n, k), poses=nan_f32(n, k, 4, 4))
    ro = lambda x, cnt: _lib.GpRansacOut(x["M"].data_ptr(), x["failed"].data_ptr(), x["in_src"].data_ptr(),
                                         x["in_tar"].data_ptr(), x["in_sc"].data_ptr(), cnt)
    pred = _lib.GpPredictions(_matches_struct(o), o["relScale"].data_ptr(), o["relInplane"].data_ptr(), ro(o, None),
                              o["scores"].data_ptr(), o["poses"].data_ptr())
    check(_lib_().gp_sort_and_pose(eng._h, b0, n, sort, qK.data_ptr(), qM.data_ptr(), C.byref(_matches_struct(m)),
                                   rel_scale.data_ptr(), rel_inplane.data_ptr(), C.byref(ro(r, r["count"].data_ptr())),
                                   C.byref(pred), _stream()))
    torch.cuda.synchronize(DEV)
    return {kk: v.cpu() for kk, v in o.items()}


def run_pose_recover(q_obj, qK, qM, id_src, M, inp, T):
    B, k = id_src.shape
    d = lambda t: t.to(DEV).contiguous()
    args = [d(q_obj.int()), d(qK), d(qM), d(id_src), d(M), d(inp["tK"]), d(inp["tM"]), d(inp["tP"])]
    poses = nan_f32(B, k, 4, 4)
    check(_lib_().gp_pose_recover(B, k, T, *(a.data_ptr() for a in args), poses.data_ptr(), _stream()))
    torch.cuda.synchronize(DEV)
    return poses.cpu()


@pytest.mark.parametrize("sort", [1, 0], ids=["sorted", "unsorted"])
def test_sort_and_pose_permutes_every_tensor_stably(sort):
    """gp_sort_and_pose at k = 32 on the window [2, 5) of 6 detections over three objects, with inlier counts drawn
    from {0, 5, 9, 256} (many equal): the order is the stable descending order (sort_by_inliers = 1) or the identity (0),
    every [B,k,...] output is a gather of its input bit for bit, scores = count / 256 exactly, and pred_poses match
    the fp64 pose lifting of the gathered hypotheses."""
    O, T, Bt, k, b0, n = 3, 40, 6, 32, 2, 3
    q_obj = torch.tensor([0, 2, 1, 2, 0, 1], dtype=torch.int32)
    inp = _pose_inputs(O, T, n, k, seed=70)
    eng = _pose_engine(O, T, Bt, k, q_obj, inp)
    g = torch.Generator().manual_seed(71)
    ri = lambda *s: torch.randint(-1, 16, s, generator=g)
    m = dict(id_src=torch.randint(0, T, (n, k), generator=g), score_src=torch.rand(n, k, generator=g),
             score_pts=torch.rand(n, k, P, generator=g), tar_pts=ri(n, k, P, 2), src_pts=ri(n, k, P, 2))
    rel_scale, rel_inplane = torch.randn(n, k, P, generator=g), torch.randn(n, k, P, 2, generator=g)
    cnt = torch.tensor([0, 5, 9, 256])[torch.randint(0, 4, (n, k), generator=g)].int()
    r = dict(M=inp["M"], failed=torch.randint(0, 2, (n, k), generator=g).to(torch.uint8), in_src=ri(n, k, P, 2),
             in_tar=ri(n, k, P, 2), in_sc=torch.randint(0, 2, (n, k, P), generator=g), count=cnt)
    d = lambda x: {kk: v.to(DEV).contiguous() for kk, v in x.items()}
    md, rd = d(m), d(r)
    out = run_sort_and_pose(eng, b0, n, sort, inp["qK"].to(DEV), inp["qM"].to(DEV), md, rel_scale.to(DEV),
                            rel_inplane.to(DEV), rd)
    order = torch.tensor([sorted(range(k), key=lambda i: -int(cnt[b, i])) if sort else list(range(k))
                          for b in range(n)])
    assert len(set(cnt[0].tolist())) < k
    gat = lambda x: torch.stack([x[b, order[b]] for b in range(n)])
    same = lambda a, b: torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))
    for key, src in (("id_src", m["id_src"]), ("score_src", m["score_src"]), ("score_pts", m["score_pts"]),
                     ("tar_pts", m["tar_pts"]), ("src_pts", m["src_pts"]), ("relScale", rel_scale),
                     ("relInplane", rel_inplane), ("M", r["M"]), ("failed", r["failed"]), ("in_src", r["in_src"]),
                     ("in_tar", r["in_tar"]), ("in_sc", r["in_sc"])):
        assert same(out[key], gat(src)), f"{key} is not the gathered input"
    assert torch.equal(out["scores"], gat(cnt).float() / 256)
    ref = pose64(q_obj[b0:b0 + n], inp["qK"], inp["qM"], gat(m["id_src"]), gat(r["M"]), inp["tK"], inp["tM"], inp["tP"])
    eR, eT, bottom = pose_err(out["poses"], ref)
    write_report(f"tail_sort_and_pose_{'sorted' if sort else 'unsorted'}.json", {"R": eR, "t": eT})
    assert bottom and eR < BAR_POSE_R and eT < BAR_POSE_T, f"rotation {eR:.3e}, translation {eT:.3e}"


def test_pose_lifting_against_fp64():
    """gp_pose_recover and gp_sort_and_pose (sort_by_inliers = 0) lift the same 8 x 10 hypotheses; both against an fp64
    restatement of port.pose_recovery.  The error is absolute on R and relative to max(|t|, 1) on the translation."""
    O, T, B, k = 2, 30, 8, 10
    inp = _pose_inputs(O, T, B, k, seed=80)
    g = torch.Generator().manual_seed(81)
    q_obj = torch.randint(0, O, (B,), generator=g).int()
    id_src = torch.randint(0, T, (B, k), generator=g)
    ref = pose64(q_obj, inp["qK"], inp["qM"], id_src, inp["M"], inp["tK"], inp["tM"], inp["tP"])
    got_pr = run_pose_recover(q_obj, inp["qK"], inp["qM"], id_src, inp["M"], inp, T)
    eng = _pose_engine(O, T, B, k, q_obj, inp)
    z = lambda *s, dt=torch.float32: torch.zeros(s, dtype=dt, device=DEV)
    md = dict(id_src=id_src.to(DEV), score_src=z(B, k), score_pts=z(B, k, P), tar_pts=z(B, k, P, 2, dt=torch.int64),
              src_pts=z(B, k, P, 2, dt=torch.int64))
    rd = dict(M=inp["M"].to(DEV), failed=z(B, k, dt=torch.uint8), in_src=z(B, k, P, 2, dt=torch.int64),
              in_tar=z(B, k, P, 2, dt=torch.int64), in_sc=z(B, k, P, dt=torch.int64), count=z(B, k, dt=torch.int32))
    out = run_sort_and_pose(eng, 0, B, 0, inp["qK"].to(DEV), inp["qM"].to(DEV), md, z(B, k, P), z(B, k, P, 2), rd)
    report = {}
    for name, got in (("pose_recover", got_pr), ("sort_and_pose", out["poses"])):
        eR, eT, bottom = pose_err(got, ref)
        report[name] = {"R": eR, "t": eT}
        assert bottom and eR < BAR_POSE_R and eT < BAR_POSE_T, f"{name}: rotation {eR:.3e}, translation {eT:.3e}"
    report["bit_identical"] = bool(torch.equal(bits(got_pr), bits(out["poses"])))
    write_report("tail_pose_lifting.json", report)
