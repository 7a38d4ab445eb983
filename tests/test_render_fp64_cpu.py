"""The renderer's contract against an fp64 ray caster (tests/render_fp64.py) without a GPU: the numpy restatement of the
kernels (oracle/render_port.py for gp_render_templates, oracle/bop_port.render_depth for gp_render_depth), which
tests/test_gpu_render.py and tests/test_gpu_bop_eval.py hold bit-identical to them, on small images of the same
scenes.  tests/test_gpu_render_fp64.py runs the same comparisons on the kernels at full size.

The bars, per sample (their derivations are in the docstring of tests/render_fp64.py):
  coverage   equal to fp64 wherever every face's score min_k E_k / dE_k lies outside [-1, 1], i.e. the sample is
             farther than delta = dE_k / |edge| (the snap plus the float32 projection error, about 1/256 px) from
             the edges that decide it;
  face       the fp64 nearest hit wherever it covers robustly and its depth interval [z - bar, z + bar] lies before
             that of every other face that may cover the sample (the depth gap exceeds both bars);
  depth      |z - z_fp64| <= S_z + c_z ulp(z): S_z the snap sensitivity, c_z = 8 + r / u (8 roundings in
             sample_weights and sample_depth, plus the float32 error r of the vertex z); and the arithmetic alone,
             |z - z_snapped| <= c_z ulp(z) against the fp64 plane through the snapped screen vertices;
  depth map  gp_render_depth: the sample's z within the depth bar, exactly 0 where fp64 says background;
             gp_render_templates: the smallest covered key, and within the bar of the fp64 smallest covered z;
  rgb        the 8-bit q within [255 c - 1/2 - e, 255 c + 1/2 + e] wherever all four samples are unambiguous, c the
             fp64 mean, e = 255 x the mean of the samples' colour bars (snap sensitivity of the attribute, through
             the texture's local Lipschitz constant for a texture, plus its float32 arithmetic) + 1e-4 for the
             resolve; a constant colour exactly;
  alpha      exact wherever one sample covers robustly or all four miss robustly;
  box        between the box of the surely covered and the box of the possibly covered pixels, and within one pixel
             of the fp64 box.
Every scene also bounds the excluded fractions (render_fp64.MAX_EXCLUDED) so that no comparison is vacuous, and six
mutated definitions must each fail clearly on the same renderer output."""
import json

import numpy as np
import pytest

from oracle import bop_port
from oracle import render_port as rp

import render_fp64 as rf

SCENES = rf.scenes(full=False)
_OUT, _CASTS = {}, {}


def _port(name):
    if name not in _OUT:
        s, m, outs = SCENES[name], SCENES[name]["mesh"], []
        for P in s["poses"]:
            if s["mode"] == "templates":
                o = rp.render(m["vertices"], m["faces"], P, s["K"], s["H"], s["W"], s["z_near"],
                              vertex_color=m.get("vertex_color"), face_uv=m.get("face_uv"), texture=m.get("texture"),
                              constant_color=m.get("constant_color"))
                outs.append(dict(keys=o["keys"], depth=o["depth"], box=o["box"], rgba=o["rgba"]))
            else:
                o = bop_port.render_depth(m["vertices"], m["faces"], P, s["K"], s["H"], s["W"], s["z_near"])
                outs.append(dict(depth=o["depth"], box=o["box"]))
        _OUT[name] = outs
    return _OUT[name]


@pytest.mark.parametrize("name", list(SCENES))
def test_port_matches_the_fp64_ray_caster_within_the_bars(name):
    rep, casts = rf.check_scene(SCENES[name], _port(name), cache=_CASTS)
    print("fp64-cpu", name, json.dumps(rep))
    rf.assert_within_bars(name, rep)
    if name.startswith("clipped"):
        rf.clipped_scene_is_exercised(SCENES[name], casts)


@pytest.mark.parametrize("mutation,name,which", rf.MUTATION_CASES)
def test_a_mutated_definition_fails_clearly(mutation, name, which):
    rep, _ = rf.check_scene(SCENES[name], _port(name), mutation, cache=_CASTS)
    n, worst = rf.assert_mutation_fails(name, mutation, rep, which)
    print("fp64-cpu-mutation", mutation, name, json.dumps(dict(fail=n, worst=worst)))


def test_the_caster_agrees_with_the_analytic_cases():
    """The caster itself on cases with a closed form: a fronto-parallel square at z = 1024 covers exactly the samples
    inside it at z = 1024; a plane tilted by 70 deg has the ray-plane depth (n . t) / (n . K^-1 (u, v, 1)); a
    texel-centred lookup returns the texel, with row 0 on top, also 3 periods and -2 periods away."""
    K = np.array([[512, 0, 0], [0, 512, 0], [0, 0, 1]], np.float32)
    s = np.float32(1024 / 512)
    V = np.array([[10.3, 5.4, 1024], [18.3, 5.4, 1024], [18.3, 13.4, 1024], [10.3, 13.4, 1024]], np.float32)
    V[:, :2] *= s
    c = rf.cast(dict(vertices=V, faces=np.array([[0, 1, 2], [0, 3, 2]])), np.eye(4), K, 24, 32, 100.0)
    want = (c.px >= 10.3) & (c.px < 18.3) & (c.py >= 5.4) & (c.py < 13.4)
    assert np.array_equal(c.covered, want) and np.allclose(c.z[want], 1024, rtol=1e-14, atol=0)
    Vp, Fp, _ = rf.grid(1, 1, 400.0, 400.0, np.random.default_rng(0))
    P = rf.pose(rf.rot([1, 0, 0], 70.0), [0.0, 0.0, 500.0])
    c = rf.cast(dict(vertices=Vp, faces=Fp), P, K, 64, 64, 100.0, n_samples=1)
    m = c.covered
    ray = np.stack([c.px[m] / 512, c.py[m] / 512, np.ones(m.sum())], 1)
    n = P[:3, 2].astype(np.float64)                               # the plane's normal in the camera frame
    zt = (n @ P[:3, 3].astype(np.float64)) / (ray @ n)
    assert m.sum() > 100 and np.allclose(c.z[m], zt, rtol=1e-12)
    tex = rf.ramp_texture()
    th, tw = tex.shape[:2]
    cc, rr = np.array([0, 5, tw - 1]), np.array([0, 7, th - 1])
    rgb, _, _ = rf.bilinear(tex.astype(np.float64), (cc + 0.5) / tw, (th - 1 - rr + 0.5) / th)
    assert np.allclose(rgb, tex[rr, cc], atol=1e-12)
    rgb, _, _ = rf.bilinear(tex.astype(np.float64), (cc + 0.5) / tw + 3, (th - 1 - rr + 0.5) / th - 2)     # repeat
    assert np.allclose(rgb, tex[rr, cc], atol=1e-12)
