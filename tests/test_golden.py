"""Pins the CPU oracle against the reference itself: fixtures under tests/golden/*.npz are outputs of the
UNMODIFIED reference kernels run on an H100 (tests/golden/make_golden.py); this test re-runs the same op chain on
the oracle (CPU only) and compares.  Tolerances: fp32 per-Gaussian ops to fast-math rounding; integer binning
outputs equal except for splats whose ellipse grazes a tile (reference: --use_fast_math); raster at the accuracy
of the reference's packed-half blend (SURVEY fact 2)."""
import os

import numpy as np
import pytest

import oracle
from tests.golden.make_golden import CASES, PARAM_KEYS, case_inputs, matched

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def run_oracle(name):
    p, cam, hw, tile, deg, up = case_inputs(name)
    out = {}
    vis, num, ids = oracle.frustum_culling_aabb(p["cluster_origin"], p["cluster_extend"], cam["frustumplane"])
    out["cull_vis"] = vis; out["cull_ids"] = ids
    act = oracle.cull_compact_activate(deg, ids, num, cam["view"], *[p[k] for k in PARAM_KEYS])
    for k, a in zip(("act_pos", "act_scale", "act_rot", "act_color", "act_opacity"), act):
        out[k] = a
    xyz, scale, rot, color, opacity = [a.reshape(*a.shape[:-2], -1) for a in act]
    inter = oracle.project(xyz, scale, rot, cam["view"], cam["proj"], hw)
    val, _, inv = oracle.eigh_and_inv_2x2matrix_forward(inter["cov2d"])
    out.update(view_pos=inter["view_pos"], ndc=inter["ndc"], T=inter["T"], J=inter["J"], cov2d=inter["cov2d"], eig_val=val, inv_cov2d=inv)
    N = xyz.shape[1]
    sl = lambda a: np.ascontiguousarray(a[..., :N])
    out["bw_inv"] = oracle.inv_2x2matrix_backward(inv, sl(up["g_inv"]))
    out["bw_cov"] = oracle.createCov2dDirectly_backward(sl(up["g_cov"]), inter["J"], cam["view"], inter["T"])
    out["bw_T_q"], out["bw_T_s"] = oracle.createTransformMatrix_backward(sl(up["g_T"]), rot, scale)
    out["bw_mvp"] = oracle.mvp_transform_backward(sl(up["g_ndc"]), sl(up["g_view"]), cam["view"], cam["proj"], inter["view_pos"])
    vz = inter["view_pos"][:, 2]
    # the reference's tile rectangle (DESIGN.md section 7, D14) and last-tile range (Q3), so that its tables compare
    lu, rd, alloc = oracle.get_allocate_size(inter["ndc"], vz, inv, opacity, hw[0], hw[1], *tile, exact_tile_bound=False)
    out["alloc"] = alloc; out["left_up"] = lu; out["right_down"] = rd
    ranges, vals, _, keys = oracle.binning(inter["ndc"], vz, inv, opacity, None, hw, tile, fix_last=False)
    out["table_keys"] = keys; out["table_vals"] = vals; out["tile_range"] = ranges
    img, T, last, *_ = oracle.rasterize_forward(vals, ranges, inter["ndc"], inv, color, opacity, None, hw[0], hw[1], *tile)
    out["img"] = img; out["final_T"] = T; out["last"] = last
    d_img = np.zeros_like(img); d_img[..., : hw[0], : hw[1]] = up["d_img"]
    gmax = float(np.abs(d_img).max())
    b = oracle.rasterize_backward(vals, ranges, inter["ndc"], inv, color, opacity, None, T, last, d_img / gmax, None, gmax, hw[0], hw[1], *tile)
    for k, a in zip(("d_ndc", "d_cov2d_inv", "d_color", "d_opacity"), b[:4]):
        out[k] = a
    A = ids.shape[0]
    ga = [np.ascontiguousarray(g[..., :A, :]) for g in up["g_act"]]
    ab = oracle.activate_backward(deg, ids, num, cam["view"], *[p[k] for k in PARAM_KEYS], *ga)
    for k, a in zip(("ab_pos", "ab_scale", "ab_rot", "ab_sh0", "ab_shr", "ab_opacity"), ab):
        out[k] = a
    return out


@pytest.mark.parametrize("name", list(CASES))
def test_oracle_with_reference_rules_matches_reference_golden(name):
    """The oracle with the reference's binning rules (exact_tile_bound=False, fix_last=False) against the reference's own
    outputs; the oracle's defaults are the corrected rules (DESIGN.md section 7, D2 and D14)."""
    path = os.path.join(GOLD, f"{name}.npz")
    ref = dict(np.load(path))
    got = run_oracle(name)
    assert np.array_equal(ref["cull_vis"].astype(bool), got["cull_vis"]) and np.array_equal(ref["cull_ids"], got["cull_ids"])
    for k in ("act_pos", "act_scale", "act_rot", "act_color", "act_opacity", "view_pos", "ndc", "T", "J", "cov2d", "inv_cov2d", "eig_val",
              "bw_inv", "bw_cov", "bw_T_q", "bw_T_s", "bw_mvp", "ab_pos", "ab_scale", "ab_rot", "ab_sh0", "ab_shr", "ab_opacity"):
        r, o = matched(ref, got, k)
        r, o = r.astype(np.float64), o.astype(np.float64)
        scale = max(1.0, float(np.abs(r).max()))
        ok = np.abs(r - o) <= 2e-5 * scale + 2e-4 * np.abs(r)
        assert ok.mean() > 0.9999, (k, 1 - ok.mean(), np.abs(r - o).max())
    same = ref["alloc"] == got["alloc"]
    assert same.mean() > 0.995, ("alloc", 1 - same.mean())
    if same.all():
        assert np.array_equal(ref["table_keys"], got["table_keys"]) and np.array_equal(ref["table_vals"], got["table_vals"])
        assert np.array_equal(ref["tile_range"], got["tile_range"])
    d = np.abs(ref["img"] - got["img"])
    assert np.quantile(d, 0.999) < 6e-3 and d.mean() < 6e-4, (np.quantile(d, 0.999), d.mean())
    for k in ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity"):
        r, o = ref[k], got[k]
        assert np.abs(r - o).sum() / (np.abs(r).sum() + 1e-30) < 5e-2, k
