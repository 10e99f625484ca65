"""GPU end-to-end parity: render_preprocess + render (Level A, op by op) and render_view (Level B, fused)
against the oracle's full forward+backward on the same seeded scene -- image and all six parameter
gradients within 1e-4 (pixels on a step-function threshold masked, SURVEY Appendix B)."""
import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import fused, render
from litegs_b200.arguments import PipelineParams
from tests.util import PARAM_KEYS, oracle_case, scaled_err, small_scene, to_torch

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _check(img, grads, nvis, ref, frag, what):
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err_img = np.abs(img[ok] - ref["img"][ok]).max()
    assert err_img < TOL, (what, "img", err_img)
    for k in PARAM_KEYS:
        g = grads[k][..., :nvis, :]
        r = ref["grads"][k][..., :nvis, :]
        e = scaled_err(g, r)
        assert e < 2e-4, (what, k, e)


@pytest.mark.parametrize("tile,sh_degree,n,hw", [((16, 16), 3, 4000, (96, 128)), ((8, 16), 2, 4000, (96, 128)), ((8, 8), 0, 4000, (96, 128)),
                                                 # BASELINE.json configs[0] ("C1"): 10k Gaussians, 256 x 256, one view
                                                 ((8, 16), 3, 10000, (256, 256)), ((12, 16), 3, 10000, (256, 256))])
def test_level_a_and_b_match_oracle(cuda, tile, sh_degree, n, hw):
    params, aabb, cam, w, frag, ref = oracle_case(n, hw, tile, sh_degree, seed=11)
    nvis = int(ref["visible_chunk_id"].shape[0])
    pp = PipelineParams(tile_size=tile)
    wt = torch.from_numpy(w).to(cuda)

    # Level A
    P, A, C = to_torch(params, aabb, cam, cuda)
    ids, num, cx, cs, cr, col, cop = render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], P["xyz"], P["scale"], P["rot"],
                                                              P["sh_0"], P["sh_rest"], P["opacity"], None, None, pp, sh_degree)
    assert int(num.item()) == nvis and np.array_equal(ids.cpu().numpy()[:nvis], ref["visible_chunk_id"])
    img, _, _, _, prim_vis = render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * pp.cluster_size, None, None, sh_degree, hw, pp)
    (img * wt).sum().backward()
    grads = {k: P[k].grad.compacted_values.cpu().numpy() for k in PARAM_KEYS}
    _check(img.detach().cpu().numpy(), grads, nvis, ref, frag, "levelA")

    # Level B
    P2, A2, C2 = to_torch(params, aabb, cam, cuda)
    img2, _, _, _, last2 = render.render_view(A2[0], A2[1], C2["frustumplane"], C2["view"], C2["proj"], P2["xyz"], P2["scale"], P2["rot"],
                                              P2["sh_0"], P2["sh_rest"], P2["opacity"], sh_degree, hw, pp)
    (img2 * wt).sum().backward()
    grads2 = {k: P2[k].grad.compacted_values.cpu().numpy() for k in PARAM_KEYS}
    _check(img2.detach().cpu().numpy(), grads2, nvis, ref, frag, "levelB")
    # the two levels agree with each other far tighter than with the CPU
    assert np.abs(img.detach().cpu().numpy() - img2.detach().cpu().numpy()).max() < 1e-5


@pytest.mark.parametrize("hw,tile,n,scales", [((96, 128), (16, 16), 4000, (0.02, 0.08)),
                                               # 32 x 32 tiles of 8 x 8 and splats hundreds of pixels wide: long tile walks, runs
                                               # longer than the emit pass's shared-memory window
                                               ((256, 256), (8, 8), 1500, (0.05, 0.5)),
                                               ((120, 200), (8, 16), 3000, (0.01, 0.2))])
def test_fused_pairs_match_oracle_lists(cuda, hw, tile, n, scales):
    """The fused pipeline's per-tile splat lists equal the oracle's (identical order) on a seeded scene."""
    from litegs_b200 import pipeline
    params, aabb, cam = small_scene(n=n, hw=hw, seed=3, log_scale_range=scales)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile)
    from tests.util import oracle_projected
    o = oracle_projected(params, aabb, cam, hw, 3)
    ranges, pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    assert st.n_pairs == pid.shape[1]
    assert np.array_equal(st.ranges.cpu().numpy(), ranges)
    assert np.array_equal(st.sorted_pid.cpu().numpy(), pid)


def test_partially_visible_scene_dense_grads(cuda):
    """Camera inside a larger cloud: some chunks culled; dense gradients of both levels agree."""
    from litegs_b200 import scene
    hw, tile = (64, 96), (8, 16)
    p = scene.make_scene(6000, sh_degree=1, cube=3.5, seed=9, log_scale_range=(0.03, 0.1))
    cam = scene.make_camera(3, 8, hw[1], hw[0])
    params = {k: p[k] for k in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    pp = PipelineParams(tile_size=tile, sparse_grad=False)
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    out = []
    for level in ("A", "B"):
        P, A, C = to_torch(params, aabb, cam, cuda)
        if level == "A":
            ids, num, cx, cs, cr, col, cop = render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], P["xyz"], P["scale"], P["rot"],
                                                                      P["sh_0"], P["sh_rest"], P["opacity"], None, None, pp, 1)
            assert 0 < int(num.item()) < A[0].shape[1]
            img = render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * 128, None, None, 1, hw, pp)[0]
        else:
            img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                     P["sh_rest"], P["opacity"], 1, hw, pp)[0]
        (img * w).sum().backward()
        out.append((img.detach().cpu().numpy(), {k: P[k].grad.cpu().numpy() for k in PARAM_KEYS}))
    assert np.abs(out[0][0] - out[1][0]).max() < 1e-5
    for k in PARAM_KEYS:
        assert scaled_err(out[0][1][k], out[1][1][k]) < 1e-4, k


def test_empty_view_renders_black(cuda):
    """A camera looking away from everything: zero visible chunks, zero pairs, black image, zero grads."""
    from litegs_b200 import scene
    hw, tile = (64, 64), (16, 16)
    p = scene.make_scene(1000, sh_degree=0, seed=1)
    V = scene.look_at_view_matrix(np.array([0.0, 0.0, 10.0]), target=(0.0, 0.0, 20.0))
    Pm = scene.proj_matrix(hw[1], hw[0])
    cam = dict(view=V[None], proj=Pm[None], frustumplane=scene.frustum_planes(V, Pm)[None])
    params = {k: p[k] for k in PARAM_KEYS}
    P, A, C = to_torch(params, (p["cluster_origin"], p["cluster_extend"]), cam, cuda)
    pp = PipelineParams(tile_size=tile, sparse_grad=False)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], 0, hw, pp)[0]
    assert float(img.detach().abs().max()) == 0.0
    img.sum().backward()
    assert all(float(P[k].grad.abs().sum()) == 0.0 for k in PARAM_KEYS)


def test_accumulate_into_dense_buffers_equals_sum_of_views(cuda):
    """render_view(accumulate_into=...) adds each view's gradients into dense buffers inside the backward kernel;
    the result equals the sum of the per-view compacted gradients scattered to dense."""
    from litegs_b200 import scene
    from litegs_b200.dist import GradAccumulator
    hw, tile = (64, 96), (16, 16)
    p = scene.make_scene(5000, sh_degree=2, cube=2.5, seed=4, log_scale_range=(0.03, 0.1))
    params = {k: p[k] for k in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    pp = PipelineParams(tile_size=tile, sparse_grad=True)
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    P, A, _ = to_torch(params, aabb, scene.make_camera(0, 8, hw[1], hw[0]), cuda)
    acc = GradAccumulator(P)
    dense_ref = {k: torch.zeros_like(P[k]) for k in PARAM_KEYS}
    for v in (0, 3, 5):
        C = {k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 8, hw[1], hw[0]).items()}
        img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                 P["sh_rest"], P["opacity"], 2, hw, pp)[0]
        (img * w).sum().backward()
        for k in PARAM_KEYS:
            dense_ref[k] += P[k].grad.to_dense()
            P[k].grad = None
        img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                 P["sh_rest"], P["opacity"], 2, hw, pp, accumulate_into=acc.grads())[0]
        (img * w).sum().backward()
        assert all(P[k].grad is None for k in PARAM_KEYS)
    got = acc.grads()
    for k in PARAM_KEYS:
        assert scaled_err(got[k].cpu().numpy(), dense_ref[k].cpu().numpy()) < 1e-6, k


def test_render_views_streams_match_serial(cuda):
    """render_views: pipelining the views of a batch over 3 CUDA streams gives the same accumulated gradients and losses
    as running them one after the other."""
    from litegs_b200 import scene
    from litegs_b200.dist import GradAccumulator
    hw, tile = (72, 96), (8, 16)
    p = scene.make_scene(8000, sh_degree=3, cube=1.5, seed=6, log_scale_range=(0.02, 0.08))
    params = {k: p[k] for k in PARAM_KEYS}
    pp = PipelineParams(tile_size=tile)
    P, A, _ = to_torch(params, (p["cluster_origin"], p["cluster_extend"]), scene.make_camera(0, 8, hw[1], hw[0]), cuda)
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 8, hw[1], hw[0]).items()} for v in range(6)]
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    res = []
    for ns in (1, 3):
        acc = GradAccumulator(P)
        losses = render.render_views(6, lambda i: cams[i], lambda i, img: (img * w).sum() * (1.0 + 0.1 * i), A[0], A[1], P["xyz"], P["scale"],
                                     P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, hw, pp, acc.grads(), n_streams=ns)
        torch.cuda.synchronize()
        res.append(([float(x) for x in losses], {k: v.clone() for k, v in acc.grads().items()}))
    assert np.allclose(res[0][0], res[1][0], rtol=1e-6)
    for k in PARAM_KEYS:
        assert scaled_err(res[1][1][k].cpu().numpy(), res[0][1][k].cpu().numpy()) < 1e-5, k
