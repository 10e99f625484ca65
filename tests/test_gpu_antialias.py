"""The antialiased mode on the GPU: the fused path against the numpy restatement (tests/aa_oracle.py) at SH degrees 0 and 3 and
two tile shapes, the off switch, graph replay and every render_views path, the camera gradient, determinism, the integrated
alpha of one splat, and one full-size C2 view."""
import math

import numpy as np
import pytest
import torch

from litegs_b200 import pipeline, render, scene
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import fused_oracle as fo
from tests.util import (PARAM_KEYS, as_f64, deterministic, differing_tiles, restatement_mask, scaled_err, single_splat,
                        small_scene, to_torch)

pytestmark = pytest.mark.gpu


def _aa_case(n, hw, tile, deg, seed, view=0, scale_range=(0.003, 0.05)):
    """Scene with many sub-pixel splats; the loss weight is zero on the oracle's fragile pixels."""
    params, aabb, cam = small_scene(n=n, hw=hw, tile=tile, sh_degree=3, seed=seed, view=view, log_scale_range=scale_range)
    w = np.random.default_rng(seed + 100).normal(size=(1, 3, hw[0], hw[1])).astype(np.float32)
    o0 = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=True)
    return params, aabb, cam, w, o0


def _forward(P, A, C, deg, hw, tile, antialiased):
    with torch.no_grad():
        return pipeline.render_view_forward({k: P[k].detach() for k in PARAM_KEYS}, A[0], A[1], C["frustumplane"], C["view"], C["proj"],
                                            deg, hw, tile, clamp_zero=True, antialiased=antialiased)


@pytest.mark.parametrize("deg,tile", [(0, (8, 16)), (0, (16, 16)), (3, (8, 16)), (3, (16, 16))])
def test_fused_path_matches_oracle(cuda, deg, tile):
    hw = (96, 128)
    params, aabb, cam, w, o0 = _aa_case(4000, hw, tile, deg, seed=11)
    assert o0["rho"][o0["rho"] > 0].min() < 0.2                       # the mode is exercised
    P, A, C = to_torch(params, aabb, cam, cuda)
    _, st, _ = _forward(P, A, C, deg, hw, tile, True)
    D = o0["sorted_pid"].shape[1]
    frag = restatement_mask(st, o0, hw, tile)
    print(f"AA deg {deg} tile {tile}: {D} pairs (ours {st.n_pairs})")
    assert abs(st.n_pairs - D) <= max(2, 1e-4 * D)
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=True)
    pp = PipelineParams(tile_size=tile, antialiased=True)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], deg, hw, pp)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err = np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max()
    assert err < 1e-4, err
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k in PARAM_KEYS:
        g = P[k].grad.compacted_values.cpu().numpy()[..., :nvis, :]
        e = scaled_err(g, ref["grads"][k][..., :nvis, :])
        print(f"  {k}: {e:.2e} of the maximum")
        assert e < 1e-4, (k, e)


def test_off_is_the_default_bit_for_bit(cuda, deterministic):
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=3, log_scale_range=(0.003, 0.05))
    w = torch.from_numpy(np.random.default_rng(1).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    outs = []
    for kw in ({}, {"antialiased": False}, {"antialiased": True}):
        P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True, **kw)
        d = torch.zeros_like(img)
        d[..., :hw[0], :hw[1]] = w
        grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img)
        outs.append([img, st.T, st.last, *grads])
    for a, b in zip(outs[0], outs[1]):
        assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], outs[2][0])


def test_deterministic_backward_and_pair_count(cuda, deterministic):
    """Two antialiased runs give the same bits; the antialiased lists are shorter (opacities only go down)."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=4, log_scale_range=(0.003, 0.05))
    w = torch.from_numpy(np.random.default_rng(2).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    runs = []
    for _ in range(2):
        P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                                  antialiased=True)
        d = torch.zeros_like(img)
        d[..., :hw[0], :hw[1]] = w
        grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img)
        runs.append([img, *grads])
        n_aa = st.n_pairs
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    _, st0, _ = _forward(P, A, C, 3, hw, tile, False)
    assert n_aa < st0.n_pairs


@pytest.mark.parametrize("std_px", [0.35, 0.7, 1.5, 3.0])
def test_integrated_alpha_on_the_gpu(cuda, std_px):
    hw = (64, 64)
    params, aabb, cam = single_splat(std_px, hw, chunk=32, dt=np.float32)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    _, st, _ = _forward(P, A, C, 0, hw, (16, 16), True)
    got = float((1 - st.T[..., :hw[0], :hw[1]]).double().sum())
    o = 0.8
    rho = std_px ** 2 / (std_px ** 2 + 0.3)
    want = 2 * math.pi * o * std_px ** 2 * (1 - 1 / (256 * o * rho))
    print(f"GPU integrated alpha at {std_px} px: {got:.5f}, predicted {want:.5f} ({(got / want - 1) * 100:+.3f} %)")
    assert abs(got / want - 1) < 0.01


def _setup_views(cuda, n=8000, hw=(72, 96), seed=6):
    p = scene.make_scene(n, sh_degree=3, cube=1.5, seed=seed, log_scale_range=(0.005, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    return P, A, cams, w


def _direct(P, A, C, hw, tile, w, antialiased, accumulate_into=None, camera_grad=None):
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              antialiased=antialiased)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    pipeline.render_view_backward(P, st, d, accumulate_into=accumulate_into, clamped_img=img, camera_grad=camera_grad)
    return img


def test_workspace_graph_replay_follows_the_mode(cuda, deterministic):
    """ViewWorkspace with graphs equals the synchronising path with the mode on, also after batches with it off in between."""
    hw, tile = (70, 100), (8, 16)
    P, A, cams, w = _setup_views(cuda, hw=hw)
    pairs, _ = pipeline.probe_view_sizes(P, A[0], A[1], cams, 3, hw, tile)
    pairs_aa, _ = pipeline.probe_view_sizes(P, A[0], A[1], cams, 3, hw, tile, antialiased=True)
    assert pairs_aa < pairs
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=int(pairs * 1.3), planned_depth_bits=32, use_graphs=True)
    acc, ref = GradAccumulator(P), GradAccumulator(P)
    side = torch.cuda.Stream(device=cuda)
    with torch.cuda.stream(side):
        for rnd in range(4):
            for aa_on in (True, False, True):
                for v in (0, 5):
                    ref.zero_(); acc.zero_()
                    cg_want = torch.empty((2, 4, 4), device=cuda)
                    img_want = _direct(P, A, cams[v], hw, tile, w, aa_on, ref.grads(), cg_want).clone()
                    img = ws.forward(P, A[0], A[1], cams[v], 3, antialiased=aa_on)
                    cg = torch.full((2, 4, 4), float("nan"), device=cuda)
                    ws.backward(P, w, 3, acc.grads(), camera_grad=cg, antialiased=aa_on)
                    side.synchronize()
                    assert torch.equal(img, img_want), (rnd, aa_on, v)
                    assert torch.equal(cg, cg_want), (rnd, aa_on, v)
                    for k in PARAM_KEYS:
                        assert torch.equal(acc.grads()[k], ref.grads()[k]), (rnd, aa_on, v, k)
    fwd = [k for k in ws._graphs if k[0] == "fwd"]
    assert any(k[1][-1] for k in fwd) and any(not k[1][-1] for k in fwd)


def _views_batch(P, A, cams, w, hw, pp, acc, views, n_streams, direct=True):
    acc.zero_()
    cg = torch.full((len(views), 2, 4, 4), float("nan"), device=w.device)
    loss_fn = lambda i, img: (img * w).sum() * (1.0 + 0.1 * views[i])
    keep = render._DIRECT_VIEWS
    try:
        render._DIRECT_VIEWS = direct
        render.render_views(len(views), lambda i: cams[views[i]], loss_fn, A[0], A[1], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                            P["sh_rest"], P["opacity"], 3, hw, pp, acc.grads(), n_streams=n_streams, camera_grads=cg)
    finally:
        render._DIRECT_VIEWS = keep
    torch.cuda.synchronize()
    return cg.clone(), {k: v.clone() for k, v in acc.grads().items()}


@pytest.mark.parametrize("n_streams", [1, 3])
def test_render_views_paths_agree(cuda, deterministic, n_streams):
    """With pp.antialiased the direct, autograd and workspace (eager, captured, replayed) paths of render_views agree bit for
    bit, and alternating batches with the mode off do not disturb them (separate capacities and graphs)."""
    hw, tile = (72, 96), (8, 16)
    P, A, cams, w = _setup_views(cuda, hw=hw)
    on, off = PipelineParams(tile_size=tile, antialiased=True), PipelineParams(tile_size=tile)
    acc = GradAccumulator(P)
    va = [0, 1, 2, 3, 4, 5]
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    try:
        pipeline.SYNC_FREE = False
        want = _views_batch(P, A, cams, w, hw, on, acc, va, n_streams)
        want_off = _views_batch(P, A, cams, w, hw, off, acc, va, n_streams)
        got = _views_batch(P, A, cams, w, hw, on, acc, va, n_streams, direct=False)
        assert torch.equal(got[0], want[0])
        for k in PARAM_KEYS:
            assert torch.equal(got[1][k], want[1][k]), k
        assert not torch.equal(want_off[0], want[0])
        pipeline.SYNC_FREE = True
        for pp, ref in ((on, want), (off, want_off), (on, want), (off, want_off), (on, want), (on, want), (off, want_off), (on, want)):
            got = _views_batch(P, A, cams, w, hw, pp, acc, va, n_streams)
            assert torch.equal(got[0], ref[0]), pp.antialiased
            for k in PARAM_KEYS:
                assert torch.equal(got[1][k], ref[1][k]), (pp.antialiased, k)
        render.check_views(wait=True)
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


@pytest.mark.parametrize("deg,view", [(3, 0), (0, 5)])
def test_camera_gradient_matches_oracle(cuda, deterministic, deg, view):
    """The camera gradient with the mode on against aa_oracle.camera_backward (which matches fp64 central differences,
    test_oracle_antialias.py), on a scene whose tile lists agree with the oracle's."""
    hw, tile = (96, 128), (16, 16)
    params, aabb, cam, w, o0 = _aa_case(4000, hw, tile, deg, seed=12, view=view)
    frag = o0["fragile"][:, :hw[0], :hw[1]]
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=True)
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, hw)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    _, st, _ = _forward(P, A, C, deg, hw, tile, True)
    bad, _ = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), ref["ranges"], ref["sorted_pid"])
    assert len(bad) == 0
    cg = torch.empty((2, 4, 4), device=cuda)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, hw, tile, clamp_zero=True,
                                              antialiased=True)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = torch.from_numpy(w).to(cuda)
    pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg)
    ev = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    ep = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"AA camera gradient vs oracle (deg {deg}, view {view}): d_view {ev:.2e}, d_proj {ep:.2e} of their maximum")
    assert ev < 1e-4 and ep < 1e-4


def test_c2_translation_identity(cuda, deterministic):
    """C2 with the mode on: sum_i d xyz_i = V3x3 . d_view[3,:3] (the rho term moves Sigma2, not the mean, so it cancels)."""
    H, W = 1080, 1920
    hw, tile = (H, W), (8, 16)
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(3, 64, W, H).items()}
    w = torch.randn((1, 3, H, W), generator=torch.Generator(device="cpu").manual_seed(4)).to(cuda)
    acc = GradAccumulator(P)
    acc.zero_()
    cg = torch.empty((2, 4, 4), device=cuda)
    _direct(P, A, C, hw, tile, w, True, acc.grads(), cg)
    gx = acc.grads()["xyz"].double().reshape(3, -1)
    s = gx.sum(dim=1).cpu().numpy()
    mag = gx.abs().sum(dim=1).cpu().numpy()
    rhs = C["view"][0, :3, :3].double().cpu().numpy() @ cg[0, 3, :3].double().cpu().numpy()
    err = np.abs(s - rhs) / mag
    print(f"C2 AA translation identity: error / sum|d xyz| {err}")
    assert np.all(err < 1e-5)


def test_c2_one_view_matches_oracle(cuda):
    """One full-size view (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles) with the mode on against the oracle, as
    test_gpu_fullsize.test_c2_one_view_matches_oracle does with it off."""
    H, W, tile, deg = 1080, 1920, (8, 16), 3
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0)
    params = {k: p[k] for k in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    cam = scene.make_camera(0, 64, W, H)
    w = np.random.default_rng(7).normal(size=(1, 3, H, W)).astype(np.float32)
    o0 = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, antialiased=True)
    frag = o0["fragile"][:, :H, :W].copy()
    assert frag.mean() < 0.10
    P, A, C = to_torch(params, aabb, cam, cuda)
    _, st, _ = _forward(P, A, C, deg, (H, W), tile, True)
    D = o0["sorted_pid"].shape[1]
    bad, npairs = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), o0["ranges"], o0["sorted_pid"])
    print(f"C2 AA view: D = {D} pairs (ours {st.n_pairs}), {len(bad)} tiles / {npairs} pairs differ, {frag.mean() * 100:.2f} % fragile")
    assert abs(st.n_pairs - D) <= 1e-5 * D and npairs <= 1e-5 * D
    gx = -(-W // tile[1])
    for t in bad:
        ty, tx = divmod(int(t), gx)
        frag[:, ty * tile[0]:(ty + 1) * tile[0], tx * tile[1]:(tx + 1) * tile[1]] = True
    lc = st.last.cpu().numpy()[:, 0, :H, :W].astype(np.uint16)
    lo = o0["last"][:, 0, :H, :W].astype(np.uint16)
    n_diff = int((lc[~frag] != lo[~frag]).sum())
    # As in test_gpu_tile_grid: after ~700 listed splats the two sides' transmittances differ by a few 1e-4 of T, wider than the
    # oracle's own margin on the 1/8192 stop; a pixel whose final T, on either side, lies within 5e-4 of it counts as fragile.
    on_stop = lambda T: np.abs(T[:, 0, :H, :W] * 8192.0 - 1.0) < 5e-4
    frag |= on_stop(st.T.cpu().numpy()) | on_stop(o0["T"])
    print(f"C2 AA view: {n_diff} contributor counts differ off the oracle's fragile pixels, all within 5e-4 of the stop: "
          f"{int((lc[~frag] != lo[~frag]).sum()) == 0}; {frag.mean() * 100:.2f} % fragile in all")
    assert np.array_equal(lc[~frag], lo[~frag])
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, antialiased=True)
    pp = PipelineParams(tile_size=tile, antialiased=True)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], deg, (H, W), pp)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err = np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max()
    assert err < 1e-4, err
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k in PARAM_KEYS:
        e = scaled_err(P[k].grad.compacted_values.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
        print(f"  {k}: {e:.2e} of the maximum")
        assert e < 2e-4, (k, e)


def test_level_a_refuses_the_mode(cuda):
    hw, tile = (48, 64), (8, 16)
    params, aabb, cam = small_scene(n=500, hw=hw, tile=tile, seed=1)
    P, A, C = to_torch(params, aabb, cam, cuda)
    pp = PipelineParams(tile_size=tile, antialiased=True)
    ids, num, cx, cs, cr, col, cop = render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], P["xyz"], P["scale"], P["rot"],
                                                              P["sh_0"], P["sh_rest"], P["opacity"], None, None, pp, 3)
    with pytest.raises(RuntimeError, match="antialiased"):
        render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * pp.cluster_size, None, None, 3, hw, pp)
