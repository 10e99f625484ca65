"""The normal mode on the GPU: normal_rec, the facing signs, N, the six gradients and the camera gradient against the numpy
restatement (tests/normal_oracle.py) at SH degrees 0 and 3, two tile shapes, the antialiased mode and the 3D filter off and on, with
depth off and on; the flag absent and off bit for bit; a zero normal gradient changes nothing (default and deterministic mode); the
direct, loss-and-grad, autograd and graph-replayed paths; the deterministic and statistics modes; the C2 translation identity; the
refusals; the workspace's gradient plane."""
import types

import numpy as np
import pytest
import torch

from litegs_b200 import _lib, pipeline, render, scene
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import filter3d_oracle as f3
from tests import fused_oracle as fo
from tests.util import (PARAM_KEYS, as_f64, deterministic, differing_tiles, lattice_cameras, restatement_mask, scaled_err,
                        small_scene, to_torch)

pytestmark = pytest.mark.gpu


def _weights(hw, seed):
    rng = np.random.default_rng(seed)
    return (rng.normal(size=(1, 3, *hw)).astype(np.float32), rng.normal(size=(1, 3, *hw)).astype(np.float32),
            rng.normal(size=(1, 1, *hw)).astype(np.float32))


CASES = [(deg, tile, aa, f) for deg in (0, 3) for tile in ((8, 16), (16, 16)) for aa in (False, True) for f in (False, True)]


@pytest.mark.parametrize("deg,tile,antialiased,filtered", CASES)
def test_fused_path_matches_restatement(cuda, deg, tile, antialiased, filtered):
    """normal_rec and sigma, the contributor counts, N (1e-4), the six gradients and the camera gradient (1e-4 of the restatement's
    maximum) with a colour and a normal loss; depth and a depth loss are on in half of the cases."""
    hw = (96, 128)
    depth = (deg == 3) == antialiased
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, sh_degree=3, seed=40 + deg, log_scale_range=(0.003, 0.05))
    filt = f3.compute_filter(params["xyz"], *lattice_cameras(24, (36, 48)))[None] if filtered else None
    if filtered:
        aabb = scene.cluster_aabb(params["xyz"], params["scale"], params["rot"], filter_3d=filt)
    w, u, uz = _weights(hw, deg)
    kw = dict(antialiased=antialiased, filter_3d=filt, render_depth=depth)
    o0 = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, render_normal=True, **kw)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    F = None if filt is None else torch.from_numpy(filt).to(cuda)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, hw, tile, clamp_zero=True,
                                              antialiased=antialiased, filter_3d=F, render_depth=depth, render_normal=True)
    # the per-record normals: visible slots against the restatement, the rest zero
    nvis = int(o0["visible_chunk_id"].shape[0])
    S = params["xyz"].shape[-1]
    rec = st.normal_rec.cpu().numpy()
    fr = o0["frame"]
    v = o0["inter"]["view_pos"][0, :3]
    dot = (fr["nc"] * v).sum(0)
    clear = np.abs(dot) > 1e-4 * np.linalg.norm(v, axis=0)          # facing decisions rounding cannot flip
    sg_gpu = np.where((rec[:nvis * S, :3] * fr["nc"].T).sum(1) < 0, -1, 1)
    assert clear.sum() > 0.9 * clear.size and np.array_equal(sg_gpu[clear], fr["sg"][clear])
    errs = {"normal_rec": np.abs(rec[:nvis * S, :3] - fr["n"].T)[clear].max()}
    assert not np.any(rec[:, 3]) and not np.any(rec[nvis * S:])
    frag = restatement_mask(st, o0, hw, tile)
    ok = ~frag[:, None]
    ok3 = np.broadcast_to(ok, o0["normal"].shape)
    errs["N"] = np.abs(st.normal.cpu().numpy()[..., :hw[0], :hw[1]] - o0["normal"])[ok3].max()
    w, u, uz = w * ok, u * ok, uz * ok
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, render_normal=True,
                                     d_normal_fn=lambda N, T: (u, None), d_depth_fn=(lambda D, T: (uz, None)) if depth else None, **kw)
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, hw, sh_degree=deg)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = torch.from_numpy(w).to(cuda)
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg, d_normal=torch.from_numpy(u).to(cuda),
                                             d_depth=torch.from_numpy(uz).to(cuda) if depth else None)
    for k, g in zip(PARAM_KEYS, grads):
        errs[k] = scaled_err(g.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
    errs["d_view"] = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    errs["d_proj"] = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"normal deg {deg} tile {tile} aa {antialiased} filter {filtered} depth {depth}: "
          + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e < 1e-4, (k, e)


def _render_grads(cuda, params, aabb, cam, hw, tile, pp, deg=3, u=None):
    """render_view + backward (a colour loss, plus sum u N when u is given) with the matrices as leaves -> dict of outputs."""
    P, A, C = to_torch(params, aabb, cam, cuda)
    view, proj = C["view"].clone().requires_grad_(True), C["proj"].clone().requires_grad_(True)
    img, _, _, normal, last = render.render_view(A[0], A[1], C["frustumplane"], view, proj, P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                                 P["sh_rest"], P["opacity"], deg, hw, pp)
    w = torch.from_numpy(np.random.default_rng(5).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    loss = (img * w).sum()
    if u is not None:
        loss = loss + (normal * u).sum()
    loss.backward()
    return dict(img=img.detach(), last=last, **{k: P[k].grad for k in PARAM_KEYS}, view=view.grad, proj=proj.grad), normal


@pytest.mark.parametrize("det", [False, True])
def test_off_and_absent_are_the_default_and_a_zero_normal_gradient_changes_nothing(cuda, det):
    """The field absent and the flag off give the same bits and no normal; with the flag on and d_normal = 0 every output and every
    gradient is the flag-off one: bit for bit in the deterministic mode; in the default mode (fp32 atomics, whose order varies from
    run to run) the forward bit for bit and the gradients within 1e-6 of their maximum.  A normal loss changes the gradients."""
    _lib.call("lgs_set_deterministic", int(det))
    try:
        hw, tile = (96, 128), (16, 16)
        params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=3, log_scale_range=(0.003, 0.05))
        fields = dict(cluster_size=128, tile_size=tile, sparse_grad=False, enable_transmitance=False, enable_depth=False)
        absent, n0 = _render_grads(cuda, params, aabb, cam, hw, tile, types.SimpleNamespace(**fields))
        off, n1 = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(**fields))
        assert n0 is None and n1 is None
        zero, nz = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(render_normal=True, **fields),
                                 u=torch.zeros((1, 3, *hw), device=cuda))
        assert nz is not None and nz.shape == (1, 3, *hw) and nz.abs().max() > 0.1
        u = torch.from_numpy(np.random.default_rng(9).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
        on, _ = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(render_normal=True, **fields), u=u)
        for k in absent:
            if det or k in ("img", "last"):
                assert torch.equal(absent[k], off[k]), k
                assert torch.equal(zero[k], off[k]), k
            else:
                assert scaled_err(absent[k].cpu().numpy(), off[k].cpu().numpy()) < 1e-6, k
                assert scaled_err(zero[k].cpu().numpy(), off[k].cpu().numpy()) < 1e-6, k
        for k in ("rot", "opacity", "view"):
            assert not torch.equal(on[k], off[k]), k
    finally:
        _lib.call("lgs_set_deterministic", 0)


def _setup_views(cuda, n=8000, hw=(72, 96), seed=6):
    p = scene.make_scene(n, sh_degree=3, cube=1.5, seed=seed, log_scale_range=(0.005, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    g = np.random.default_rng(0)
    w = torch.from_numpy(g.normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    u = torch.from_numpy(g.normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    uz = torch.from_numpy(g.normal(size=(1, 1, *hw)).astype(np.float32)).to(cuda)
    return P, A, cams, w, u, uz


def _views_batch(P, A, cams, w, u, uz, hw, pp, acc, views, n_streams, direct=True, grad_fn=False):
    """One render_views batch; with the normal flag the loss is colour + sum u EN over the covered pixels (d_trans included), plus
    sum uz D with the depth flag."""
    acc.zero_()
    cg = torch.full((len(views), 2, 4, 4), float("nan"), device=w.device)
    nrm, dep = getattr(pp, "render_normal", False), getattr(pp, "render_depth", False)
    if not nrm and not dep:
        loss_fn, lg = (lambda i, img: (img * w).sum() * (1.0 + 0.1 * views[i])), None
    else:
        def loss_fn(i, img, depth, trans, normal=None):
            a = 1 - trans
            loss = (img * w).sum()
            if normal is not None:
                loss = loss + (torch.where(a > 0.2, normal / a.clamp_min(0.2), torch.zeros_like(normal)) * u).sum()
            if depth is not None:
                loss = loss + (depth * uz).sum()
            return loss * (1.0 + 0.1 * views[i])

        def lg(i, img, depth, trans, *normal):
            ins = [img, depth, trans, *normal]
            leaves = [None if t is None else t.detach().requires_grad_(True) for t in ins]
            loss = loss_fn(i, *leaves)
            live = [t for t in leaves if t is not None]
            gs = iter(torch.autograd.grad(loss, live))
            return (loss, *(None if t is None else next(gs) for t in leaves))
    keep = render._DIRECT_VIEWS
    try:
        render._DIRECT_VIEWS = direct
        render.render_views(len(views), lambda i: cams[views[i]], None if grad_fn and lg else loss_fn, A[0], A[1], P["xyz"], P["scale"],
                            P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, hw, pp, acc.grads(), n_streams=n_streams, camera_grads=cg,
                            loss_and_grad_fn=lg if grad_fn else None)
    finally:
        render._DIRECT_VIEWS = keep
    torch.cuda.synchronize()
    return cg.clone(), {k: v.clone() for k, v in acc.grads().items()}


@pytest.mark.parametrize("n_streams", [1, 3])
def test_render_views_paths_agree(cuda, deterministic, n_streams):
    """With an expected-normal loss (so d_trans as well) the direct, loss_and_grad_fn, autograd and workspace (eager, captured,
    replayed) paths agree bit for bit, with depth off and on, also when the flags alternate between batches."""
    hw, tile = (72, 96), (8, 16)
    P, A, cams, w, u, uz = _setup_views(cuda, hw=hw)
    pp_n, pp_nd = PipelineParams(tile_size=tile, render_normal=True), PipelineParams(tile_size=tile, render_normal=True, render_depth=True)
    pp_off = PipelineParams(tile_size=tile)
    acc = GradAccumulator(P)
    va = [0, 1, 2, 3, 4, 5]
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    same = lambda a, b: torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in PARAM_KEYS)
    try:
        pipeline.SYNC_FREE = False
        want = {id(pp): _views_batch(P, A, cams, w, u, uz, hw, pp, acc, va, n_streams) for pp in (pp_n, pp_nd, pp_off)}
        assert not torch.equal(want[id(pp_off)][1]["rot"], want[id(pp_n)][1]["rot"])
        assert not torch.equal(want[id(pp_nd)][1]["xyz"], want[id(pp_n)][1]["xyz"])
        for pp in (pp_n, pp_nd):
            assert same(_views_batch(P, A, cams, w, u, uz, hw, pp, acc, va, n_streams, grad_fn=True), want[id(pp)])
            assert same(_views_batch(P, A, cams, w, u, uz, hw, pp, acc, va, n_streams, direct=False), want[id(pp)])
        pipeline.SYNC_FREE = True
        for pp in (pp_n, pp_off, pp_n, pp_nd, pp_n, pp_nd, pp_off, pp_nd, pp_n):
            assert same(_views_batch(P, A, cams, w, u, uz, hw, pp, acc, va, n_streams), want[id(pp)]), (pp.render_normal, pp.render_depth)
        assert same(_views_batch(P, A, cams, w, u, uz, hw, pp_nd, acc, va, n_streams, grad_fn=True), want[id(pp_nd)])
        render.check_views(wait=True)
        ws = next(iter(render._slot_cache.values())).ws[0]
        seen = set(ws._graphs) | set(ws._eager_runs)
        assert len([k for k in seen if k[0] == "fwd"]) == 3 and len([k for k in seen if k[0] == "bwd"]) == 3
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


def _one_view(cuda, P, A, C, hw, tile, u, w, stat=False, acc=None, exact=False):
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              enable_statistic=stat, render_normal=True)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, pg = pipeline.render_view_backward(P, st, d, enable_statistic=stat, accumulate_into=acc, clamped_img=img, camera_grad=cg,
                                              exact_grad=exact, d_normal=u)
    return st.normal.clone(), grads, cg, pg


def test_deterministic_and_statistics_modes(cuda, deterministic):
    """Deterministic mode: two runs with normals give the same bits.  Statistics on (13 reduced values, 2 parked splats per flush):
    N, the gradients and the camera gradient equal the statistics-off run to 1e-6 of their maximum."""
    hw, tile = (96, 128), (16, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=11, log_scale_range=(0.003, 0.05))
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    w, u, _ = (torch.from_numpy(x).to(cuda) for x in _weights(hw, 1))
    a = _one_view(cuda, P, A, C, hw, tile, u, w)
    b = _one_view(cuda, P, A, C, hw, tile, u, w)
    s = _one_view(cuda, P, A, C, hw, tile, u, w, stat=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x, y)
    errs = {"N": scaled_err(s[0].cpu().numpy(), a[0].cpu().numpy()), "cam": scaled_err(s[2].cpu().numpy(), a[2].cpu().numpy())}
    for k, x, y in zip(PARAM_KEYS, s[1], a[1]):
        errs[k] = scaled_err(x.cpu().numpy(), y.cpu().numpy())
    print("statistics on vs off with normals: " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e < 1e-6, (k, e)


@pytest.mark.parametrize("exact", [False, True])
def test_c2_translation_identity_with_a_normal_loss(cuda, exact):
    """C2 (1M Gaussians, 1920x1080, SH degree 3) with a colour and a normal loss: sum_i d xyz_i = V3x3 . d_view[3,:3] within 1e-5
    of sum |d xyz|, in the default convention and in the exact mode."""
    H, W = 1080, 1920
    hw, tile = (H, W), (8, 16)
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(3, 64, W, H).items()}
    g = torch.Generator(device="cpu").manual_seed(4)
    w, u = torch.randn((1, 3, H, W), generator=g).to(cuda), torch.randn((1, 3, H, W), generator=g).to(cuda)
    acc = GradAccumulator(P)
    acc.zero_()
    _, _, cg, _ = _one_view(cuda, P, A, C, hw, tile, u, w, acc=acc.grads(), exact=exact)
    gx = acc.grads()["xyz"].double().reshape(3, -1)
    s = gx.sum(dim=1).cpu().numpy()
    mag = gx.abs().sum(dim=1).cpu().numpy()
    rhs = C["view"][0, :3, :3].double().cpu().numpy() @ cg[0, 3, :3].double().cpu().numpy()
    err = np.abs(s - rhs) / mag
    print(f"C2 translation identity with normals, exact={exact}: error / sum|d xyz| {err}")
    assert np.all(err < 1e-5)


def test_refusals(cuda):
    """Normals exist on the default raster kernels only (the pixel-pair forward, bulk staging and the scalar backward refuse them);
    Level A's render() refuses the flag; d_normal after a forward without normals is refused by the pipeline and the workspace."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=2000, hw=hw, tile=tile, seed=2)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    fwd = lambda: pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                               render_normal=True)
    img, st, _ = fwd()
    d, u = torch.ones_like(img), torch.ones((1, 3, *hw), device=cuda)
    try:
        _lib.call("lgs_set_forward_pairs", 1)
        with pytest.raises(RuntimeError, match="pixel-pair forward"):
            fwd()
        _lib.call("lgs_set_forward_pairs", 0)
        _lib.call("lgs_set_staging", 1)
        with pytest.raises(RuntimeError, match="bulk staging"):
            fwd()
        with pytest.raises(RuntimeError, match="bulk staging"):
            pipeline.render_view_backward(P, st, d, clamped_img=img, d_normal=u)
        _lib.call("lgs_set_staging", 0)
        _lib.call("lgs_set_backward_kernel", 1)
        with pytest.raises(RuntimeError, match="scalar"):
            pipeline.render_view_backward(P, st, d, clamped_img=img, d_normal=u)
    finally:
        _lib.call("lgs_set_forward_pairs", 0)
        _lib.call("lgs_set_staging", 0)
        _lib.call("lgs_set_backward_kernel", 2)
    pipeline.render_view_backward(P, st, d, clamped_img=img, d_normal=u)
    _, st0, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True)
    with pytest.raises(RuntimeError, match="did not render normals"):
        pipeline.render_view_backward(P, st0, d, clamped_img=img, d_normal=u)
    pp = PipelineParams(tile_size=tile, render_normal=True)
    with pytest.raises(RuntimeError, match="render_normal"):
        render.render(*([None] * 12), pp)
    Pd = {k: v.detach() for k, v in P.items()}
    ws = pipeline.ViewWorkspace(Pd, hw, tile, pair_capacity=1 << 20, use_graphs=False)
    acc = GradAccumulator(Pd)
    ws.forward(Pd, A[0], A[1], C, 3)
    with pytest.raises(RuntimeError, match="did not render normals"):
        ws.backward(Pd, d[..., :hw[0], :hw[1]], 3, acc.grads(), d_normal=u)


def test_workspace_clears_stale_normal_gradient_padding(cuda, deterministic):
    """hw not a multiple of the tile: the workspace's d_normal plane is zeroed in the padding before an [H,W] gradient is copied in,
    so a stale padded [Hp,Wp] gradient of an earlier call does not leak into the next backward."""
    hw, tile = (90, 120), (16, 16)
    params, aabb, cam = small_scene(n=3000, hw=hw, tile=tile, seed=8)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1 << 20, use_graphs=False)
    acc = GradAccumulator(P)
    w = torch.randn((1, 3, *hw), device=cuda)
    u = torch.randn((1, 3, *hw), device=cuda)

    def run(du):
        acc.zero_()
        ws.forward(P, A[0], A[1], C, 3, render_normal=True)
        ws.backward(P, w, 3, acc.grads(), d_normal=du)
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in acc.grads().items()}

    ref = run(u)
    junk = torch.full((1, 3, ws.Hp, ws.Wp), 1e3, device=cuda)
    junk[..., :hw[0], :hw[1]] = u
    run(junk)                                                        # fills the padding of the plane with 1e3
    got = run(u)
    assert ws.d_normal[..., hw[0]:, :].abs().max() == 0 and ws.d_normal[..., hw[1]:].abs().max() == 0
    for k in PARAM_KEYS:
        assert torch.equal(got[k], ref[k]), k


def test_train_colmap_normal_weight_lowers_the_normal_error(cuda, tmp_path):
    """examples/train_colmap.py --normal-weight on a small synthetic dataset (make_dataset writes the hidden scene's unit normals):
    the GPU-driven path trains with the term, and the mean angle to the target normals ends lower than in the same run without it;
    with --depth-weight as well, both terms train together."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("train_colmap", os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples",
                                                                              "train_colmap.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    root = mod.make_dataset(str(tmp_path / "ds"), n_gaussians=8000, n_views=8, hw=(96, 160), n_points=4000, dev=cuda)
    assert len(os.listdir(os.path.join(root, "normals"))) == 8
    res = {}
    for wn, wd in ((0.0, 0.0), (0.3, 0.0), (0.3, 0.3)):
        m = {}
        hist, psnr = mod.train(root, iters=120, views_per_step=4, log=lambda *_: None, normal_weight=wn, depth_weight=wd, metrics=m)
        res[(wn, wd)] = (hist, psnr, m["normal_angle"])
    print("train_colmap: " + ", ".join(f"normal/depth weight {k}: loss {v[0][0]:.4f} -> {v[0][-1]:.4f}, PSNR {v[1]:.2f} dB, "
                                       f"normal angle {v[2]:.2f} deg" for k, v in res.items()))
    for k in ((0.3, 0.0), (0.3, 0.3)):
        assert res[k][0][-1] < res[k][0][0]
        assert res[k][2] < res[(0.0, 0.0)][2]


def test_chunk_sizes_beyond_the_normal_kernels_limits_are_refused(cuda):
    """The NORMAL instantiations need more registers than the default ones, so they launch fewer threads per block.  Chunks the
    default kernels take but a NORMAL one cannot launch are refused with the limit named, before any launch:
    project_forward with the antialiased mode and the 3D filter at SH degree 3 (56 -> 72 registers: 1024 -> 896 threads) at
    chunks of 1024, and project_backward at SH degree 3 (96 -> 124 registers: 672 -> 512 threads) at chunks of 640."""
    hw, tile = (72, 96), (8, 16)
    for chunk, where in ((1024, "project_forward"), (640, "project_backward")):
        p = scene.make_scene(6000, sh_degree=3, chunk=chunk, seed=2, log_scale_range=(0.005, 0.05))
        P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
        A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
        C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(0, 8, hw[1], hw[0]).items()}
        aa = where == "project_forward"
        F = torch.zeros_like(P["opacity"]) if aa else None      # a zero filter selects the F3D kernels and changes no scale
        fwd = lambda nrm: pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile,
                                                       clamp_zero=True, antialiased=aa, filter_3d=F, render_normal=nrm)
        img, st, _ = fwd(False)
        assert st.n_chunks_visible > 0
        if where == "project_forward":
            with pytest.raises(RuntimeError, match=r"project_forward: normals with this configuration support chunk sizes up to "
                                                   r"[0-9]+, got 1024"):
                fwd(True)
        else:
            pipeline.render_view_backward(P, st, torch.ones_like(img), clamped_img=img)
            img, st, _ = fwd(True)
            pipeline.render_view_backward(P, st, torch.ones_like(img), clamped_img=img)      # normals rendered, no normal loss
            with pytest.raises(RuntimeError, match=r"project_backward: the normal gradient with this configuration supports chunk "
                                                   r"sizes up to [0-9]+, got 640"):
                pipeline.render_view_backward(P, st, torch.ones_like(img), clamped_img=img, d_normal=torch.ones((1, 3, *hw), device=cuda))


def test_c2_one_view_matches_restatement(cuda):
    """One full-size view (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles) with a colour, a normal and a depth loss against the
    restatement: N, the image, the six gradients and the camera gradient, fragile pixels excluded as in test_gpu_depth.py.  The
    few Gaussians whose facing decision sits within rounding of zero take the GPU's sign in the restatement."""
    H, W, tile, deg = 1080, 1920, (8, 16), 3
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0)
    params = {k: p[k] for k in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    cam = scene.make_camera(0, 64, W, H)
    g = np.random.default_rng(7)
    w, u, uz = (g.normal(size=(1, 3, H, W)).astype(np.float32), g.normal(size=(1, 3, H, W)).astype(np.float32),
                g.normal(size=(1, 1, H, W)).astype(np.float32))
    o0 = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, render_normal=True, render_depth=True)
    frag = o0["fragile"][:, :H, :W].copy()
    assert frag.mean() < 0.10
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, (H, W), tile, clamp_zero=True,
                                              render_depth=True, render_normal=True)
    bad, npairs = differing_tiles(st.ranges.cpu().numpy(), st.sorted_pid.cpu().numpy(), o0["ranges"], o0["sorted_pid"])
    D = o0["sorted_pid"].shape[1]
    assert abs(st.n_pairs - D) <= 1e-5 * D and npairs <= 1e-5 * D
    gx = -(-W // tile[1])
    for t in bad:
        ty, tx = divmod(int(t), gx)
        frag[:, ty * tile[0]:(ty + 1) * tile[0], tx * tile[1]:(tx + 1) * tile[1]] = True
    on_stop = lambda T: np.abs(T[:, 0, :H, :W] * 8192.0 - 1.0) < 5e-4          # as test_gpu_antialias's C2 view
    frag |= on_stop(st.T.cpu().numpy()) | on_stop(o0["T"])
    lc, lo = st.last.cpu().numpy()[:, 0, :H, :W].astype(np.uint16), o0["last"][:, 0, :H, :W].astype(np.uint16)
    assert np.array_equal(lc[~frag], lo[~frag])
    # facing signs: equal wherever rounding cannot flip them; the restatement then uses the GPU's signs throughout
    nvis = int(o0["visible_chunk_id"].shape[0])
    S = params["xyz"].shape[-1]
    fr = o0["frame"]
    rec = st.normal_rec.cpu().numpy()[:nvis * S, :3]
    sg_gpu = np.where((rec * fr["nc"].T).sum(1) < 0, -1, 1).astype(np.float32)
    v = o0["inter"]["view_pos"][0, :3]
    clear = np.abs((fr["nc"] * v).sum(0)) > 1e-4 * np.linalg.norm(v, axis=0)
    assert np.array_equal(sg_gpu[clear], fr["sg"][clear])
    freeze = dict(a=fr["a"], sg=sg_gpu)
    ok = ~frag[:, None]
    w, u, uz = w * ok, u * ok, uz * ok
    ref = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, render_normal=True, render_depth=True,
                                     d_normal_fn=lambda N_, T_: (u, None), d_depth_fn=lambda D_, T_: (uz, None), normal_freeze=freeze)
    ok3 = np.broadcast_to(ok, ref["normal"].shape)
    errs = {"img": np.abs(img.cpu().numpy()[..., :H, :W] - ref["img"])[np.broadcast_to(ok, ref["img"].shape)].max(),
            "normal_rec": np.abs(rec - ref["frame"]["n"].T).max(),
            "N": np.abs(st.normal.cpu().numpy()[..., :H, :W] - ref["normal"])[ok3].max(),
            "D": np.abs(st.depth.cpu().numpy()[..., :H, :W] - ref["depth"])[ok].max() / np.abs(ref["depth"]).max()}
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, (H, W), sh_degree=deg)
    d = torch.zeros_like(img)
    d[..., :H, :W] = torch.from_numpy(w).to(cuda)
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg, d_normal=torch.from_numpy(u).to(cuda),
                                             d_depth=torch.from_numpy(uz).to(cuda))
    for k, gr in zip(PARAM_KEYS, grads):
        errs[k] = scaled_err(gr.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
    errs["d_view"] = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    errs["d_proj"] = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"C2 normal view ({frag.mean() * 100:.2f} % fragile, {int((~clear).sum())} of {clear.size} facing decisions within "
          f"rounding of zero, {int((sg_gpu != fr['sg']).sum())} differing): " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    assert errs.pop("img") < 1e-4
    assert errs.pop("normal_rec") < 1e-5
    for k, e in errs.items():
        assert e < 2e-4, (k, e)
