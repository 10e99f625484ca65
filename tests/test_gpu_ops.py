"""GPU parity tests (H100): every op of the C ABI, through the litegs_fused-shaped host mirror, against
the CPU oracle on identical seeded inputs.  Integer/index outputs must be bit-exact; fp32 outputs within
1e-4 relative (BASELINE.json north_star); pixels the oracle flags as sitting on a step-function
threshold (SURVEY Appendix B) are masked and counted."""
import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import fused
from tests.util import oracle_projected, rel_err, scaled_err, small_scene

pytestmark = pytest.mark.gpu
TOL = 1e-4


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def proj(cuda):
    hw = (96, 128)
    params, aabb, cam = small_scene(n=3000, hw=hw)
    o = oracle_projected(params, aabb, cam, hw, 3)
    return dict(params=params, aabb=aabb, cam=cam, hw=hw, o=o)


def test_frustum_culling_and_activate(cuda, proj):
    p, aabb, cam = proj["params"], proj["aabb"], proj["cam"]
    # move the camera so that some chunks are culled
    cam2 = dict(cam)
    vis, num, ids = fused.frustum_culling_aabb(T(aabb[0], cuda), T(aabb[1], cuda), T(cam["frustumplane"], cuda), None, None)
    ovis, onum, oids = oracle.frustum_culling_aabb(aabb[0], aabb[1], cam["frustumplane"])
    assert int(num.item()) == int(onum[0])
    assert np.array_equal(vis.cpu().numpy(), ovis)
    assert np.array_equal(ids.cpu().numpy(), oids)
    out = fused.cull_compact_activate(3, ids, num, T(cam["view"], cuda), *[T(p[k], cuda) for k in ("xyz", "scale", "rot", "sh_0", "sh_rest", "opacity")])
    ref = proj["o"]["act"]
    for a, b, name in zip(out, ref, ("pos", "scale", "rot", "color", "opacity")):
        assert rel_err(a.cpu().numpy(), b) < TOL, name


def test_partial_visibility_ordered_compaction(cuda):
    from litegs_b200 import scene
    p = scene.make_scene(20000, sh_degree=1, cube=4.0, seed=5)
    cam = scene.make_camera(2, 8, 128, 96)
    vis, num, ids = fused.frustum_culling_aabb(T(p["cluster_origin"], cuda), T(p["cluster_extend"], cuda), T(cam["frustumplane"], cuda), None, None)
    ovis, onum, oids = oracle.frustum_culling_aabb(p["cluster_origin"], p["cluster_extend"], cam["frustumplane"])
    assert 0 < int(onum[0]) < p["cluster_origin"].shape[1]
    assert np.array_equal(ids.cpu().numpy(), oids) and np.array_equal(vis.cpu().numpy(), ovis)


def test_projection_ops_forward_backward(cuda, proj):
    o, cam, hw = proj["o"], proj["cam"], proj["hw"]
    view, pm = T(cam["view"], cuda), T(cam["proj"], cuda)
    vp, ndc = fused.mvp_transform_forward(T(o["xyz"], cuda), view, pm, None)
    assert rel_err(vp.cpu().numpy(), o["view_pos"]) < TOL and rel_err(ndc.cpu().numpy(), o["ndc"]) < TOL
    Tm = fused.createTransformMatrix_forward(T(o["rot"], cuda), T(o["scale"], cuda), None)
    assert rel_err(Tm.cpu().numpy(), o["T"]) < TOL
    J = fused.jacobianRayspace(T(o["view_pos"], cuda), pm, hw[0], hw[1], None)
    assert scaled_err(J.cpu().numpy(), o["J"]) < TOL
    cov = fused.createCov2dDirectly_forward(T(o["J"], cuda), view, T(o["T"], cuda), None)
    assert rel_err(cov.cpu().numpy(), o["cov2d"]) < TOL
    val, vec, inv = fused.eigh_and_inv_2x2matrix_forward(T(o["cov2d"], cuda), None)
    oval, ovec, oinv = oracle.eigh_and_inv_2x2matrix_forward(o["cov2d"])
    assert rel_err(inv.cpu().numpy(), oinv) < TOL and rel_err(val.cpu().numpy(), oval) < TOL
    # backward chain with random upstream gradients
    rng = np.random.default_rng(0)
    N = o["xyz"].shape[1]
    g_inv = rng.normal(size=(1, 2, 2, N)).astype(np.float32)
    g_inv[:, 1, 0] = g_inv[:, 0, 1]
    a = fused.inv_2x2matrix_backward(T(oinv, cuda), T(g_inv, cuda), None).cpu().numpy()
    b = oracle.inv_2x2matrix_backward(oinv, g_inv)
    assert scaled_err(a, b) < TOL
    g_cov = rng.normal(size=(1, 2, 2, N)).astype(np.float32)
    g_cov[:, 1, 0] = g_cov[:, 0, 1]
    a = fused.createCov2dDirectly_backward(T(g_cov, cuda), T(o["J"], cuda), view, T(o["T"], cuda), None).cpu().numpy()
    b = oracle.createCov2dDirectly_backward(g_cov, o["J"], cam["view"], o["T"])
    assert scaled_err(a, b) < TOL
    gT = rng.normal(size=(3, 3, N)).astype(np.float32)
    gq, gs = fused.createTransformMatrix_backward(T(gT, cuda), T(o["rot"], cuda), T(o["scale"], cuda), None)
    oq, os_ = oracle.createTransformMatrix_backward(gT, o["rot"], o["scale"])
    assert scaled_err(gq.cpu().numpy(), oq) < TOL and scaled_err(gs.cpu().numpy(), os_) < TOL
    gn = rng.normal(size=(1, 4, N)).astype(np.float32); gv = rng.normal(size=(1, 4, N)).astype(np.float32)
    a = fused.mvp_transform_backward(T(gn, cuda), T(gv, cuda), view, pm, T(o["view_pos"], cuda), None).cpu().numpy()
    b = oracle.mvp_transform_backward(gn, gv, cam["view"], cam["proj"], o["view_pos"])
    assert scaled_err(a, b) < TOL


def test_valid_length_is_respected(cuda, proj):
    o, cam = proj["o"], proj["cam"]
    N = o["xyz"].shape[1]
    vl = torch.tensor([N // 2], dtype=torch.int32, device=cuda)
    _, _, al = fused.get_allocate_size(T(o["ndc"], cuda), T(o["view_pos"][:, 2], cuda), T(o["inv_cov2d"], cuda), T(o["opacity"], cuda),
                                       proj["hw"][0], proj["hw"][1], 16, 16, vl)
    _, _, oal = oracle.get_allocate_size(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], proj["hw"][0], proj["hw"][1], 16, 16,
                                         np.array([N // 2], np.int32))
    assert np.array_equal(al.cpu().numpy(), oal) and int(al[:, N // 2:].abs().sum()) == 0


@pytest.mark.parametrize("tile", [(16, 16), (8, 16), (12, 16), (8, 8)])
def test_binning_bit_exact(cuda, proj, tile):
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ndc, vz, inv, op = (T(o["ndc"], cuda), T(o["view_pos"][:, 2].copy(), cuda), T(o["inv_cov2d"], cuda), T(o["opacity"], cuda))
    lu, rd, al = fused.get_allocate_size(ndc, vz, inv, op, hw[0], hw[1], th, tw, None)
    olu, ord_, oal = oracle.get_allocate_size(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], hw[0], hw[1], th, tw)
    assert np.array_equal(al.cpu().numpy(), oal)
    assert np.array_equal(lu.cpu().numpy(), olu) and np.array_equal(rd.cpu().numpy(), ord_)
    # wrapper.py:739-745 in torch, then our create_table / tileRange
    order = np.argsort(o["view_pos"][:, 2], axis=-1, kind="stable").astype(np.int64)
    prefix = np.cumsum(np.take_along_axis(oal, order, -1), -1).astype(np.int32)
    keys, vals = fused.create_table(ndc, inv, op, T(prefix, cuda), T(order, cuda), None, None, hw[0], hw[1], th, tw)
    okeys, ovals = oracle.create_table(o["ndc"], o["inv_cov2d"], o["opacity"], prefix, order, int(prefix[0, -1]), hw[0], hw[1], th, tw)
    assert np.array_equal(keys.cpu().numpy(), okeys) and np.array_equal(vals.cpu().numpy(), ovals)
    gx, gy = (hw[1] + tw - 1) // tw, (hw[0] + th - 1) // th
    rng_ = fused.tileRange(keys, gx * gy)
    assert np.array_equal(rng_.cpu().numpy(), oracle.tileRange(okeys, gx * gy, fix_last=True))


def _raster_case(cuda, proj, tile, staging):
    from litegs_b200 import _lib
    _lib.call("lgs_set_staging", 1 if staging == "bulk" else 0)
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, sorted_pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    oimg, oT, olast, _, _, fragile = oracle.rasterize_forward(sorted_pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None,
                                                               hw[0], hw[1], th, tw, fragile_eps=2e-6)
    out = fused.rasterize_forward(T(sorted_pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                  T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, False, False, False)
    img, Tr, _, last, packed, _, _ = out
    ok = ~fragile
    assert fragile.mean() < 0.02
    assert np.array_equal(last.cpu().numpy()[:, 0][ok], olast[:, 0][ok])
    m3 = np.broadcast_to(ok[:, None], oimg.shape)
    assert rel_err(img.cpu().numpy()[m3], oimg[m3]) < TOL
    assert rel_err(Tr.cpu().numpy()[:, 0][ok], oT[:, 0][ok]) < TOL
    # backward, fed with the ORACLE's forward state so that only the backward kernel is under test
    rng = np.random.default_rng(1)
    g = rng.normal(size=oimg.shape).astype(np.float32)
    g[np.broadcast_to(fragile[:, None], g.shape)] = 0.0
    gmax = np.abs(g).max()
    ref = oracle.rasterize_backward(sorted_pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast,
                                    g / gmax, None, gmax, hw[0], hw[1], th, tw)
    got = fused.rasterize_backward(T(sorted_pid, cuda), T(ranges, cuda), packed, None, T(oT, cuda), T(olast, cuda), T(g / gmax, cuda),
                                   None, None, torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, False)
    for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
        assert scaled_err(a.cpu().numpy(), b) < TOL, (name, scaled_err(a.cpu().numpy(), b))


@pytest.mark.parametrize("staging", ["bulk", "cpasync"])
@pytest.mark.parametrize("tile", [(16, 16), (8, 16), (12, 16), (8, 8)])
def test_raster_forward_backward(cuda, proj, tile, staging):
    _raster_case(cuda, proj, tile, staging)
