"""Mip-Splatting's 3D smoothing filter on the GPU: lgs_filter_3d against the numpy restatement (tests/filter3d_oracle.py) bit for
bit, the fused path with a filter against the restatement at SH degrees 0 and 3, two tile shapes and the antialiased mode off and
on, the no-filter and zero-filter identities, graph replay and every render_views path, the camera gradient, determinism, one
full-size C2 view and a short training run."""
import os

import numpy as np
import pytest
import torch

from litegs_b200 import pipeline, render, scene
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import filter3d_oracle as f3
from tests import fused_oracle as fo
from tests.util import (PARAM_KEYS, as_f64, deterministic, differing_tiles, lattice_cameras, restatement_mask, scaled_err,
                        small_scene, to_torch)

pytestmark = pytest.mark.gpu


def _device_filter(xyz, views, projs, hws, cuda, out=None):
    return scene.filter_3d_device(torch.from_numpy(np.ascontiguousarray(xyz)).to(cuda), torch.from_numpy(views).to(cuda),
                                  torch.from_numpy(projs).to(cuda), torch.from_numpy(hws).to(cuda), out=out)


def _kernel_cases():
    rng = np.random.default_rng(0)
    xyz = scene.cluster(rng.uniform(-1.5, 1.5, (3, 5000)).astype(np.float32), 128)
    # the cameras below sit on the upper half of the lattice sphere and look at the origin: the first four chunks, moved to
    # y = 80 above them, are behind or far outside every one of them
    far = xyz.copy()
    far[:, :4] *= 0.1
    far[1, :4] += 80.0
    mixed_v, mixed_p, mixed_hw = [], [], []
    for i, (w, h, fov) in enumerate([(64, 48, 60.0), (200, 90, 40.0), (33, 77, 85.0), (512, 512, 20.0)]):
        c = scene.make_camera(i, 8, w, h, fov_x_deg=fov)
        mixed_v.append(c["view"]); mixed_p.append(c["proj"]); mixed_hw.append((h, w))
    mixed = (np.concatenate(mixed_v), np.concatenate(mixed_p), np.array(mixed_hw, np.int32))
    v1 = lattice_cameras(1, (90, 160))
    # the camera at z = -3 looks towards -z: every point is behind it
    cam_behind = (np.stack([scene.look_at_view_matrix(np.array([0.0, 0.0, -3.0]), target=(0.0, 0.0, -10.0))]),
                  scene.proj_matrix(64, 64)[None], np.array([[64, 64]], np.int32))
    return {"V=1": (xyz, *v1), "V=1000": (far, *(x[:1000] for x in lattice_cameras(2000, (72, 96)))), "mixed sizes": (far, *mixed),
            "none seen": (xyz, *cam_behind)}


@pytest.mark.parametrize("case", ["V=1", "V=1000", "mixed sizes", "none seen"])
def test_filter_kernel_matches_restatement_bit_for_bit(cuda, case):
    xyz, views, projs, hws = _kernel_cases()[case]
    want = f3.compute_filter(xyz, views, projs, hws)
    got = _device_filter(xyz, views, projs, hws, cuda)
    again = _device_filter(xyz, views, projs, hws, cuda)
    assert got.shape == (1, *xyz.shape[-2:])
    g = got.cpu().numpy()[0]
    n_bad = int((g.view(np.uint32) != want.view(np.uint32)).sum())
    print(f"{case}: {n_bad} of {g.size} differ, f in [{want.min():.3e}, {want.max():.3e}]")
    assert n_bad == 0
    assert torch.equal(got, again)
    if case == "none seen":
        assert np.all(want == 0)
    if case in ("V=1000", "mixed sizes"):
        assert np.sum(want == want.max()) >= 4 * 128                  # the unseen chunks carry the largest seen value


def _case(n, hw, tile, deg, seed, antialiased, view=0, scale_range=(0.003, 0.05)):
    """Scene with sub-pixel splats and a filter from 24 low-resolution lattice cameras, strong enough that rho3 < 0.5 occurs."""
    params, aabb, cam = small_scene(n=n, hw=hw, tile=tile, sh_degree=3, seed=seed, view=view, log_scale_range=scale_range)
    filt = f3.compute_filter(params["xyz"], *lattice_cameras(24, (36, 48)))[None]
    aabb = scene.cluster_aabb(params["xyz"], params["scale"], params["rot"], filter_3d=filt)
    w = np.random.default_rng(seed + 100).normal(size=(1, 3, hw[0], hw[1])).astype(np.float32)
    o0 = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=antialiased, filter_3d=filt)
    return params, aabb, cam, filt, w, o0


def _forward(P, A, C, deg, hw, tile, antialiased, filt):
    with torch.no_grad():
        return pipeline.render_view_forward({k: P[k].detach() for k in PARAM_KEYS}, A[0], A[1], C["frustumplane"], C["view"], C["proj"],
                                            deg, hw, tile, clamp_zero=True, antialiased=antialiased, filter_3d=filt)


@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("deg,tile", [(0, (8, 16)), (0, (16, 16)), (3, (8, 16)), (3, (16, 16))])
def test_fused_path_matches_oracle(cuda, deg, tile, antialiased):
    hw = (96, 128)
    params, aabb, cam, filt, w, o0 = _case(4000, hw, tile, deg, 11, antialiased)
    assert o0["rho3"].min() < 0.5
    P, A, C = to_torch(params, aabb, cam, cuda)
    F = torch.from_numpy(filt).to(cuda)
    _, st, _ = _forward(P, A, C, deg, hw, tile, antialiased, F)
    D = o0["sorted_pid"].shape[1]
    frag = restatement_mask(st, o0, hw, tile)
    print(f"F3D aa={antialiased} deg {deg} tile {tile}: {D} pairs (ours {st.n_pairs})")
    assert abs(st.n_pairs - D) <= max(2, 1e-4 * D)
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=antialiased, filter_3d=filt)
    pp = PipelineParams(tile_size=tile, antialiased=antialiased)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], deg, hw, pp, filter_3d=F)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err = np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max()
    assert err < 1e-4, err
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k in PARAM_KEYS:
        e = scaled_err(P[k].grad.compacted_values.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
        print(f"  {k}: {e:.2e} of the maximum")
        assert e < 1e-4, (k, e)


@pytest.mark.parametrize("antialiased", [False, True])
def test_no_filter_is_the_default_and_zero_filter_is_no_filter(cuda, deterministic, antialiased):
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=3, log_scale_range=(0.003, 0.05))
    w = torch.from_numpy(np.random.default_rng(1).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    C_, S_ = params["xyz"].shape[-2:]
    zero = torch.zeros((1, C_, S_), device=cuda)
    some = torch.full((1, C_, S_), 0.01, device=cuda)
    outs = []
    for kw in ({}, {"filter_3d": None}, {"filter_3d": zero}, {"filter_3d": some}):
        P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                                  antialiased=antialiased, **kw)
        d = torch.zeros_like(img)
        d[..., :hw[0], :hw[1]] = w
        cg = torch.empty((2, 4, 4), device=cuda)
        grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg)
        outs.append([img, st.T, st.last, st.packed, cg, *grads])
    for other in outs[1:3]:
        for a, b in zip(outs[0], other):
            assert torch.equal(a, b)
    assert not torch.equal(outs[0][0], outs[3][0])


def test_deterministic_backward_and_fewer_pairs(cuda, deterministic):
    """Two filtered runs give the same bits; the filter lowers the opacities, and on this scene of sub-pixel splats the lists get
    shorter."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=4, log_scale_range=(0.003, 0.05))
    filt = torch.from_numpy(f3.compute_filter(params["xyz"], *lattice_cameras(24, (36, 48)))[None]).to(cuda)
    w = torch.from_numpy(np.random.default_rng(2).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    runs = []
    for _ in range(2):
        P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
        img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                                  filter_3d=filt)
        d = torch.zeros_like(img)
        d[..., :hw[0], :hw[1]] = w
        grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img)
        runs.append([img, *grads])
        n_f = st.n_pairs
    for a, b in zip(*runs):
        assert torch.equal(a, b)
    _, st0, _ = _forward(P, A, C, 3, hw, tile, False, None)
    print(f"pairs: {st0.n_pairs} without the filter, {n_f} with it")
    assert n_f < st0.n_pairs


def _setup_views(cuda, n=8000, hw=(72, 96), seed=6):
    p = scene.make_scene(n, sh_degree=3, cube=1.5, seed=seed, log_scale_range=(0.005, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    views, projs, hws = (torch.from_numpy(a).to(cuda) for a in lattice_cameras(12, (24, 32)))
    F = scene.filter_3d_device(P["xyz"], views, projs, hws)
    return P, A, cams, w, F, (views, projs, hws)


def _direct(P, A, C, hw, tile, w, filt, accumulate_into=None, camera_grad=None, antialiased=False):
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              antialiased=antialiased, filter_3d=filt)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    pipeline.render_view_backward(P, st, d, accumulate_into=accumulate_into, clamped_img=img, camera_grad=camera_grad)
    return img


def test_workspace_graph_replay_follows_the_filter(cuda, deterministic):
    """ViewWorkspace with graphs equals the synchronising path with the filter, with batches without it in between; recomputing the
    filter in place is seen by the replayed graphs, and a new filter tensor is captured anew."""
    hw, tile = (70, 100), (8, 16)
    P, A, cams, w, F, cam_set = _setup_views(cuda, hw=hw)
    pairs, _ = pipeline.probe_view_sizes(P, A[0], A[1], cams, 3, hw, tile)
    pairs_f, _ = pipeline.probe_view_sizes(P, A[0], A[1], cams, 3, hw, tile, filter_3d=F)
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=int(max(pairs, pairs_f) * 1.3), planned_depth_bits=32, use_graphs=True)
    acc, ref = GradAccumulator(P), GradAccumulator(P)
    side = torch.cuda.Stream(device=cuda)
    F2 = F.clone()

    def check(filt, tag):
        for v in (0, 5):
            ref.zero_(); acc.zero_()
            cg_want = torch.empty((2, 4, 4), device=cuda)
            img_want = _direct(P, A, cams[v], hw, tile, w, filt, ref.grads(), cg_want).clone()
            img = ws.forward(P, A[0], A[1], cams[v], 3, filter_3d=filt)
            cg = torch.full((2, 4, 4), float("nan"), device=cuda)
            ws.backward(P, w, 3, acc.grads(), camera_grad=cg, filter_3d=filt)
            side.synchronize()
            assert torch.equal(img, img_want), (tag, v)
            assert torch.equal(cg, cg_want), (tag, v)
            for k in PARAM_KEYS:
                assert torch.equal(acc.grads()[k], ref.grads()[k]), (tag, v, k)
            yield img.clone()

    with torch.cuda.stream(side):
        for rnd in range(3):
            for tag, filt in (("F", F), ("off", None), ("F", F)):
                imgs = list(check(filt, tag))
        n_graphs = len(ws._graphs)
        # recompute in place with other cameras: same pointer, the replayed graphs read the new values
        views, projs, hws = cam_set
        scene.filter_3d_device(P["xyz"], views[:3], projs[:3], hws[:3] * 4, out=F)
        assert not torch.equal(F, F2)
        imgs_new = list(check(F, "F recomputed"))
        assert len(ws._graphs) == n_graphs
        assert not torch.equal(imgs_new[0], imgs[0])
        # a new tensor is a new signature: eager, then captured
        for _ in range(3):
            list(check(F2, "F2"))
        assert len(ws._graphs) == n_graphs + 2
    sigs = [k[1][-2] for k in ws._graphs if k[0] == "fwd"]
    assert 0 in sigs and F.data_ptr() in sigs and F2.data_ptr() in sigs


def _views_batch(P, A, cams, w, hw, pp, acc, views, n_streams, filt, direct=True):
    acc.zero_()
    cg = torch.full((len(views), 2, 4, 4), float("nan"), device=w.device)
    loss_fn = lambda i, img: (img * w).sum() * (1.0 + 0.1 * views[i])
    keep = render._DIRECT_VIEWS
    try:
        render._DIRECT_VIEWS = direct
        render.render_views(len(views), lambda i: cams[views[i]], loss_fn, A[0], A[1], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                            P["sh_rest"], P["opacity"], 3, hw, pp, acc.grads(), n_streams=n_streams, camera_grads=cg, filter_3d=filt)
    finally:
        render._DIRECT_VIEWS = keep
    torch.cuda.synchronize()
    return cg.clone(), {k: v.clone() for k, v in acc.grads().items()}


@pytest.mark.parametrize("n_streams", [1, 3])
def test_render_views_paths_agree(cuda, deterministic, n_streams):
    """With a filter the direct, autograd and workspace (eager, captured, replayed) paths of render_views agree bit for bit, and
    batches without the filter in between do not disturb them (separate capacities and graphs)."""
    hw, tile = (72, 96), (8, 16)
    P, A, cams, w, F, _ = _setup_views(cuda, hw=hw)
    pp = PipelineParams(tile_size=tile)
    acc = GradAccumulator(P)
    va = [0, 1, 2, 3, 4, 5]
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    try:
        pipeline.SYNC_FREE = False
        want = _views_batch(P, A, cams, w, hw, pp, acc, va, n_streams, F)
        want_off = _views_batch(P, A, cams, w, hw, pp, acc, va, n_streams, None)
        got = _views_batch(P, A, cams, w, hw, pp, acc, va, n_streams, F, direct=False)
        assert torch.equal(got[0], want[0])
        for k in PARAM_KEYS:
            assert torch.equal(got[1][k], want[1][k]), k
        assert not torch.equal(want_off[0], want[0])
        pipeline.SYNC_FREE = True
        for filt, ref in ((F, want), (None, want_off), (F, want), (None, want_off), (F, want), (F, want), (None, want_off), (F, want)):
            got = _views_batch(P, A, cams, w, hw, pp, acc, va, n_streams, filt)
            assert torch.equal(got[0], ref[0]), filt is None
            for k in PARAM_KEYS:
                assert torch.equal(got[1][k], ref[1][k]), (filt is None, k)
        render.check_views(wait=True)
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


@pytest.mark.parametrize("antialiased", [False, True])
@pytest.mark.parametrize("deg,view", [(3, 0), (0, 5)])
def test_camera_gradient_matches_oracle(cuda, deterministic, deg, view, antialiased):
    hw, tile = (96, 128), (16, 16)
    params, aabb, cam, filt, w, o0 = _case(4000, hw, tile, deg, 12, antialiased, view=view)
    frag = o0["fragile"][:, :hw[0], :hw[1]]
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, antialiased=antialiased, filter_3d=filt)
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, hw)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    F = torch.from_numpy(filt).to(cuda)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, hw, tile, clamp_zero=True,
                                              antialiased=antialiased, filter_3d=F)
    bad, _ = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), ref["ranges"], ref["sorted_pid"])
    assert len(bad) == 0
    cg = torch.empty((2, 4, 4), device=cuda)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = torch.from_numpy(w).to(cuda)
    pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg)
    ev = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    ep = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"F3D camera gradient vs oracle (deg {deg}, view {view}, aa {antialiased}): d_view {ev:.2e}, d_proj {ep:.2e} of their maximum")
    assert ev < 1e-4 and ep < 1e-4


def _c2(cuda):
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    views, projs, hws = lattice_cameras(24, (1080, 1920))
    filt = f3.compute_filter(p["xyz"], views, projs, hws)[None]
    return p, filt


def test_c2_translation_identity(cuda, deterministic):
    """C2 with the filter: sum_i d xyz_i = V3x3 . d_view[3,:3] (the filter moves Sigma2 and the opacity, not the mean)."""
    H, W = 1080, 1920
    hw, tile = (H, W), (8, 16)
    p, filt = _c2(cuda)
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    F = torch.from_numpy(filt).to(cuda)
    A = [t.contiguous() for t in scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"], filter_3d=F)]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(3, 64, W, H).items()}
    w = torch.randn((1, 3, H, W), generator=torch.Generator(device="cpu").manual_seed(4)).to(cuda)
    acc = GradAccumulator(P)
    acc.zero_()
    cg = torch.empty((2, 4, 4), device=cuda)
    _direct(P, A, C, hw, tile, w, F, acc.grads(), cg)
    gx = acc.grads()["xyz"].double().reshape(3, -1)
    s = gx.sum(dim=1).cpu().numpy()
    mag = gx.abs().sum(dim=1).cpu().numpy()
    rhs = C["view"][0, :3, :3].double().cpu().numpy() @ cg[0, 3, :3].double().cpu().numpy()
    err = np.abs(s - rhs) / mag
    print(f"C2 F3D translation identity: error / sum|d xyz| {err}")
    assert np.all(err < 1e-5)


def test_c2_one_view_matches_oracle(cuda):
    """One full-size view (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles) with a filter from 24 lattice cameras against the
    restatement, as test_gpu_antialias does for its mode.  The device filter equals the restatement's bit for bit."""
    H, W, tile, deg = 1080, 1920, (8, 16), 3
    p, filt = _c2(cuda)
    params = {k: p[k] for k in PARAM_KEYS}
    got = _device_filter(p["xyz"], *lattice_cameras(24, (H, W)), cuda).cpu().numpy()
    assert np.array_equal(got.view(np.uint32), filt.view(np.uint32))
    aabb = scene.cluster_aabb(p["xyz"], p["scale"], p["rot"], filter_3d=filt)
    cam = scene.make_camera(0, 64, W, H)
    w = np.random.default_rng(7).normal(size=(1, 3, H, W)).astype(np.float32)
    o0 = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, filter_3d=filt)
    print(f"C2 filter: f in [{filt.min():.2e}, {filt.max():.2e}], rho3 min {o0['rho3'].min():.3f}, "
          f"{(o0['rho3'] < 0.9).mean() * 100:.1f} % of the visible Gaussians below 0.9")
    frag = o0["fragile"][:, :H, :W].copy()
    assert frag.mean() < 0.10
    P, A, C = to_torch(params, aabb, cam, cuda)
    F = torch.from_numpy(filt).to(cuda)
    _, st, _ = _forward(P, A, C, deg, (H, W), tile, False, F)
    D = o0["sorted_pid"].shape[1]
    bad, npairs = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), o0["ranges"], o0["sorted_pid"])
    print(f"C2 F3D view: D = {D} pairs (ours {st.n_pairs}), {len(bad)} tiles / {npairs} pairs differ, {frag.mean() * 100:.2f} % fragile")
    assert abs(st.n_pairs - D) <= 1e-5 * D and npairs <= 1e-5 * D
    gx = -(-W // tile[1])
    for t in bad:
        ty, tx = divmod(int(t), gx)
        frag[:, ty * tile[0]:(ty + 1) * tile[0], tx * tile[1]:(tx + 1) * tile[1]] = True
    lc = st.last.cpu().numpy()[:, 0, :H, :W].astype(np.uint16)
    lo = o0["last"][:, 0, :H, :W].astype(np.uint16)
    # as in test_gpu_antialias: a pixel whose final T, on either side, lies within 5e-4 of the 1/8192 stop counts as fragile
    on_stop = lambda T: np.abs(T[:, 0, :H, :W] * 8192.0 - 1.0) < 5e-4
    frag |= on_stop(st.T.cpu().numpy()) | on_stop(o0["T"])
    assert np.array_equal(lc[~frag], lo[~frag])
    w = w * (~frag)[:, None]
    ref = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, filter_3d=filt)
    pp = PipelineParams(tile_size=tile)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], deg, (H, W), pp, filter_3d=F)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err = np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max()
    assert err < 1e-4, err
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k in PARAM_KEYS:
        e = scaled_err(P[k].grad.compacted_values.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
        print(f"  {k}: {e:.2e} of the maximum")
        assert e < 2e-4, (k, e)


def test_train_colmap_with_filter(cuda, tmp_path):
    """examples/train_colmap.py --filter-3d on a small synthetic dataset: the GPU-driven workspace path runs with the filter and the
    loss falls."""
    import importlib.util
    spec = importlib.util.spec_from_file_location("train_colmap", os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples",
                                                                              "train_colmap.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    root = mod.make_dataset(str(tmp_path / "ds"), n_gaussians=8000, n_views=8, hw=(96, 160), n_points=4000, dev=cuda)
    render.reset_view_workspaces()
    try:
        hist, psnr = mod.train(root, iters=120, views_per_step=4, log=lambda *_: None, filter_3d=True)
        slots = [e for k, e in render._slot_cache.items() if k[-1]]
        assert slots and all(e.ws for e in slots)                     # the filtered configuration ran on workspaces
    finally:
        render.reset_view_workspaces()
    print(f"train_colmap --filter-3d: loss {hist[0]:.4f} -> {hist[-1]:.4f}, PSNR {psnr:.2f} dB")
    assert hist[-1] < 0.5 * hist[0] and psnr > 20.0, (hist[0], hist[-1], psnr)
