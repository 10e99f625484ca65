"""The depth mode on the GPU: D and the six gradients and the camera gradient against the numpy restatement (tests/depth_oracle.py)
at SH degrees 0 and 3, two tile shapes and the antialiased mode and the 3D filter off and on; sum w = 1 - T; the flag absent and off
bit for bit; a zero depth gradient changes nothing; the direct, autograd and graph-replayed paths; the deterministic and statistics
modes; the C2 translation identity and one C2 view against the restatement; the depth slot's own effect in project_backward; the
workspace's gradient planes; the refusal of the non-default raster variants; train_colmap --depth-weight."""
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
    return rng.normal(size=(1, 3, *hw)).astype(np.float32), rng.normal(size=(1, 1, *hw)).astype(np.float32)


CASES = [(deg, tile, aa, f) for deg in (0, 3) for tile in ((8, 16), (16, 16)) for aa in (False, True) for f in (False, True)]


@pytest.mark.parametrize("deg,tile,antialiased,filtered", CASES)
def test_fused_path_matches_restatement(cuda, deg, tile, antialiased, filtered):
    hw = (96, 128)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, sh_degree=3, seed=40 + deg, log_scale_range=(0.003, 0.05))
    filt = f3.compute_filter(params["xyz"], *lattice_cameras(24, (36, 48)))[None] if filtered else None
    if filtered:
        aabb = scene.cluster_aabb(params["xyz"], params["scale"], params["rot"], filter_3d=filt)
    w, u = _weights(hw, deg)
    kw = dict(antialiased=antialiased, filter_3d=filt)
    o0 = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, render_depth=True, **kw)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    F = None if filt is None else torch.from_numpy(filt).to(cuda)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, hw, tile, clamp_zero=True,
                                              antialiased=antialiased, filter_3d=F, render_depth=True)
    frag = restatement_mask(st, o0, hw, tile)
    ok = ~frag[:, None]
    errs = {"img": np.abs(img.cpu().numpy()[..., :hw[0], :hw[1]] - o0["img"])[np.broadcast_to(ok, o0["img"].shape)].max(),
            "D": np.abs(st.depth.cpu().numpy()[..., :hw[0], :hw[1]] - o0["depth"])[ok].max() / np.abs(o0["depth"]).max()}
    w, u = w * ok, u * ok
    ref = fo.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w, render_depth=True, d_depth_fn=lambda D, T: (u, None),
                                     **kw)
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, hw, sh_degree=deg)
    nvis = int(ref["visible_chunk_id"].shape[0])
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = torch.from_numpy(w).to(cuda)
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg, d_depth=torch.from_numpy(u).to(cuda))
    for k, g in zip(PARAM_KEYS, grads):
        errs[k] = scaled_err(g.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
    errs["d_view"] = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    errs["d_proj"] = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"depth deg {deg} tile {tile} aa {antialiased} filter {filtered}: " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e < 1e-4, (k, e)


def test_weights_sum_to_one_minus_T(cuda):
    """sum w = 1 - T on the GPU: the depth kernel fed records whose depth slot holds 1 returns 1 - T up to fp32 rounding, so
    D / (1 - T) is a weighted mean of the depths."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=3, log_scale_range=(0.003, 0.05))
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              render_depth=True)
    packed = st.packed.clone()
    packed[..., 9] = 1.0
    sw, T = torch.empty_like(st.T), torch.empty_like(st.T)
    img2, last = torch.empty_like(img), torch.empty_like(st.last)
    _lib.call("lgs_rasterize_forward_packed", pipeline._ptr(st.sorted_pid), pipeline._ptr(st.ranges), pipeline._ptr(packed), None, 0, 1,
              packed.shape[1], st.sorted_pid.shape[1], hw[0], hw[1], tile[0], tile[1], 0, 1, pipeline._ptr(img2), pipeline._ptr(T),
              pipeline._ptr(last), None, None, None, pipeline._ptr(sw), None, None, pipeline._stream(cuda))
    torch.cuda.synchronize()
    assert torch.equal(T, st.T) and torch.equal(img2, img)
    err = (sw - (1 - T)).abs().max().item()
    print(f"sum w - (1 - T): {err:.1e}")
    assert err < 1e-5
    z = st.depth / (1 - st.T).clamp_min(1e-6)
    m = (1 - st.T) > 0.5
    zk = st.packed[0, :, 9][st.tile_count > 0]
    assert z[m].min() >= zk.min() * (1 - 1e-4) and z[m].max() <= zk.max() * (1 + 1e-4)


def _render_grads(cuda, params, aabb, cam, hw, tile, pp, deg=3, u=None):
    """render_view + backward (a colour loss, plus sum u D when u is given) with the matrices as leaves -> dict of outputs."""
    P, A, C = to_torch(params, aabb, cam, cuda)
    view, proj = C["view"].clone().requires_grad_(True), C["proj"].clone().requires_grad_(True)
    img, _, depth, _, last = render.render_view(A[0], A[1], C["frustumplane"], view, proj, P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                                P["sh_rest"], P["opacity"], deg, hw, pp)
    w = torch.from_numpy(np.random.default_rng(5).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    loss = (img * w).sum()
    if u is not None:
        loss = loss + (depth * u).sum()
    loss.backward()
    return dict(img=img.detach(), last=last, **{k: P[k].grad for k in PARAM_KEYS}, view=view.grad, proj=proj.grad), depth


@pytest.mark.parametrize("antialiased", [False, True])
def test_off_and_absent_are_the_default_and_a_zero_depth_gradient_changes_nothing(cuda, deterministic, antialiased):
    """The field absent and the flag off give the same bits and no depth; with the flag on and d_depth = 0 every output and every
    gradient is the flag-off one bit for bit; with a depth loss the gradients change and d proj column 2 stays zero."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=3, log_scale_range=(0.003, 0.05))
    fields = dict(cluster_size=128, tile_size=tile, sparse_grad=False, enable_transmitance=False, enable_depth=False,
                  antialiased=antialiased)
    absent, d0 = _render_grads(cuda, params, aabb, cam, hw, tile, types.SimpleNamespace(**fields))
    off, d1 = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(**fields))
    assert d0 is None and d1 is None
    zero, dz = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(render_depth=True, **fields),
                             u=torch.zeros((1, 1, *hw), device=cuda))
    assert dz is not None and dz.shape == (1, 1, *hw) and dz.abs().max() > 1
    u = torch.from_numpy(np.random.default_rng(9).normal(size=(1, 1, *hw)).astype(np.float32)).to(cuda)
    on, _ = _render_grads(cuda, params, aabb, cam, hw, tile, PipelineParams(render_depth=True, **fields), u=u)
    for k in absent:
        assert torch.equal(absent[k], off[k]), k
        assert torch.equal(zero[k], off[k]), k
    for k in ("xyz", "scale", "opacity", "view"):
        assert not torch.equal(on[k], off[k]), k
    assert torch.equal(on["proj"][0, :, 2], off["proj"][0, :, 2])


def _setup_views(cuda, n=8000, hw=(72, 96), seed=6):
    p = scene.make_scene(n, sh_degree=3, cube=1.5, seed=seed, log_scale_range=(0.005, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    g = np.random.default_rng(0)
    w = torch.from_numpy(g.normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    u = torch.from_numpy(g.normal(size=(1, 1, *hw)).astype(np.float32)).to(cuda)
    return P, A, cams, w, u


def _views_batch(P, A, cams, w, u, hw, pp, acc, views, n_streams, direct=True, grad_fn=False):
    """One render_views batch; with the depth flag the loss is colour + sum u ED over the covered pixels (d_trans included)."""
    acc.zero_()
    cg = torch.full((len(views), 2, 4, 4), float("nan"), device=w.device)
    if not getattr(pp, "render_depth", False):
        loss_fn, lg = (lambda i, img: (img * w).sum() * (1.0 + 0.1 * views[i])), None
    else:
        def loss_fn(i, img, depth, trans):
            a = 1 - trans
            ed = torch.where(a > 0.2, depth / a.clamp_min(0.2), torch.zeros_like(depth))
            return ((img * w).sum() + (ed * u).sum()) * (1.0 + 0.1 * views[i])

        def lg(i, img, depth, trans):
            leaves = [t.detach().requires_grad_(True) for t in (img, depth, trans)]
            loss = loss_fn(i, *leaves)
            return (loss, *torch.autograd.grad(loss, leaves))
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
    """With an expected-depth loss (so d_trans as well) the direct, loss_and_grad_fn, autograd and workspace (eager, captured,
    replayed) paths of render_views agree bit for bit, also when the flag alternates between batches."""
    hw, tile = (72, 96), (8, 16)
    P, A, cams, w, u = _setup_views(cuda, hw=hw)
    pp_on, pp_off = PipelineParams(tile_size=tile, render_depth=True), PipelineParams(tile_size=tile)
    acc = GradAccumulator(P)
    va = [0, 1, 2, 3, 4, 5]
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    same = lambda a, b: torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in PARAM_KEYS)
    try:
        pipeline.SYNC_FREE = False
        want = _views_batch(P, A, cams, w, u, hw, pp_on, acc, va, n_streams)
        want_off = _views_batch(P, A, cams, w, u, hw, pp_off, acc, va, n_streams)
        assert not torch.equal(want_off[1]["xyz"], want[1]["xyz"])
        assert same(_views_batch(P, A, cams, w, u, hw, pp_on, acc, va, n_streams, grad_fn=True), want)
        assert same(_views_batch(P, A, cams, w, u, hw, pp_on, acc, va, n_streams, direct=False), want)
        pipeline.SYNC_FREE = True
        for pp, ref in ((pp_on, want), (pp_off, want_off), (pp_on, want), (pp_on, want), (pp_off, want_off), (pp_on, want),
                        (pp_off, want_off)):
            assert same(_views_batch(P, A, cams, w, u, hw, pp, acc, va, n_streams), ref), pp.render_depth
        assert same(_views_batch(P, A, cams, w, u, hw, pp_on, acc, va, n_streams, grad_fn=True), want)
        render.check_views(wait=True)
        assert len(render._slot_cache) == 1
        ws = next(iter(render._slot_cache.values())).ws[0]
        seen = set(ws._graphs) | set(ws._eager_runs)
        assert len([k for k in seen if k[0] == "fwd"]) == 2 and len([k for k in seen if k[0] == "bwd"]) == 2
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


def _one_view(cuda, P, A, C, hw, tile, u, w, stat=False, acc=None, exact=False):
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              enable_statistic=stat, render_depth=True)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, pg = pipeline.render_view_backward(P, st, d, enable_statistic=stat, accumulate_into=acc, clamped_img=img, camera_grad=cg,
                                              exact_grad=exact, d_depth=u)
    return st.depth.clone(), grads, cg, pg


def test_deterministic_and_statistics_modes(cuda, deterministic):
    """Deterministic mode: two runs with depth give the same bits.  Statistics on (11 reduced values, 2 parked splats per flush):
    D, the gradients, the camera gradient and the depth slot equal the statistics-off run to 1e-6 of their maximum."""
    hw, tile = (96, 128), (16, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=11, log_scale_range=(0.003, 0.05))
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    w, u = (torch.from_numpy(x).to(cuda) for x in _weights(hw, 1))
    a = _one_view(cuda, P, A, C, hw, tile, u, w)
    b = _one_view(cuda, P, A, C, hw, tile, u, w)
    s = _one_view(cuda, P, A, C, hw, tile, u, w, stat=True)
    assert torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]) and torch.equal(a[3], b[3])
    for x, y in zip(a[1], b[1]):
        assert torch.equal(x, y)
    assert a[3][..., 10].abs().max() > 0
    errs = {"D": scaled_err(s[0].cpu().numpy(), a[0].cpu().numpy()), "cam": scaled_err(s[2].cpu().numpy(), a[2].cpu().numpy()),
            "slot10": scaled_err(s[3][..., 10].cpu().numpy(), a[3][..., 10].cpu().numpy())}
    for k, x, y in zip(PARAM_KEYS, s[1], a[1]):
        errs[k] = scaled_err(x.cpu().numpy(), y.cpu().numpy())
    print("statistics on vs off with depth: " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    for k, e in errs.items():
        assert e < 1e-6, (k, e)


@pytest.mark.parametrize("exact", [False, True])
def test_c2_translation_identity_with_a_depth_loss(cuda, exact):
    """C2 (1M Gaussians, 1920x1080, SH degree 3) with a colour and a depth loss: sum_i d xyz_i = V3x3 . d_view[3,:3] within 1e-5
    of sum |d xyz|, in the default convention and in the exact mode."""
    H, W = 1080, 1920
    hw, tile = (H, W), (8, 16)
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(3, 64, W, H).items()}
    g = torch.Generator(device="cpu").manual_seed(4)
    w, u = torch.randn((1, 3, H, W), generator=g).to(cuda), torch.randn((1, 1, H, W), generator=g).to(cuda)
    acc = GradAccumulator(P)
    acc.zero_()
    _, _, cg, _ = _one_view(cuda, P, A, C, hw, tile, u, w, acc=acc.grads(), exact=exact)
    gx = acc.grads()["xyz"].double().reshape(3, -1)
    s = gx.sum(dim=1).cpu().numpy()
    mag = gx.abs().sum(dim=1).cpu().numpy()
    rhs = C["view"][0, :3, :3].double().cpu().numpy() @ cg[0, 3, :3].double().cpu().numpy()
    err = np.abs(s - rhs) / mag
    print(f"C2 translation identity with depth, exact={exact}: error / sum|d xyz| {err}")
    assert np.all(err < 1e-5)


def test_non_default_raster_variants_refuse_depth(cuda):
    """Depth exists on the default raster kernels only: with the pixel-pair forward, bulk staging or the scalar backward forced,
    the entry point returns an error instead of dropping the depth."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=2000, hw=hw, tile=tile, seed=2)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    fwd = lambda: pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                               render_depth=True)
    img, st, _ = fwd()
    d, u = torch.ones_like(img), torch.ones((1, 1, *hw), device=cuda)
    try:
        _lib.call("lgs_set_forward_pairs", 1)
        with pytest.raises(RuntimeError, match="pixel-pair forward"):
            fwd()
        _lib.call("lgs_set_forward_pairs", 0)
        _lib.call("lgs_set_staging", 1)
        with pytest.raises(RuntimeError, match="bulk staging"):
            fwd()
        with pytest.raises(RuntimeError, match="bulk staging"):
            pipeline.render_view_backward(P, st, d, clamped_img=img, d_depth=u)
        _lib.call("lgs_set_staging", 0)
        _lib.call("lgs_set_backward_kernel", 1)
        with pytest.raises(RuntimeError, match="scalar"):
            pipeline.render_view_backward(P, st, d, clamped_img=img, d_depth=u)
    finally:
        _lib.call("lgs_set_forward_pairs", 0)
        _lib.call("lgs_set_staging", 0)
        _lib.call("lgs_set_backward_kernel", 2)
    pipeline.render_view_backward(P, st, d, clamped_img=img, d_depth=u)
    _, st0, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True)
    with pytest.raises(RuntimeError, match="did not render depth"):
        pipeline.render_view_backward(P, st0, d, clamped_img=img, d_depth=u)


def _project(cuda, P, st, pg, depth):
    """lgs_project_backward alone on a given record gradient (compacted outputs, camera gradient) -> (grads, d_cam f32[2,4,4])."""
    C, S = P["xyz"].shape[-2:]
    A, R = st.n_chunks_visible, P["sh_rest"].shape[0]
    out = [torch.zeros((n, A, S), device=cuda) for n in (3, 3, 4)] + [torch.zeros((1, 3, A, S), device=cuda),
                                                                    torch.zeros((R, 3, A, S), device=cuda), torch.zeros((1, A, S), device=cuda)]
    part, cam = torch.empty((A, 32), device=cuda), torch.empty((2, 4, 4), device=cuda)
    p = pipeline._ptr
    _lib.call("lgs_project_backward", st.sh_degree, p(st.chunk_ids), p(st.counters), p(st.view), p(st.proj), p(P["xyz"]), p(P["scale"]),
              p(P["rot"]), p(P["opacity"]), C, S, A, R, *st.hw, 0, p(pg), None, 1, *(p(t) for t in out), None, p(part), p(cam), None, 0,
              p(P["sh_0"]), p(P["sh_rest"]), 0, int(depth), None, pipeline._stream(cuda))
    torch.cuda.synchronize()
    return out, cam


def test_depth_slot_reaches_view_column_2_and_not_proj(cuda):
    """project_backward with the depth slot read vs ignored, on the same record gradient: only d xyz and d_view column 2 change
    (by p~_k dz summed over the Gaussians, within fp32 rounding of the fp64 sum); d_proj and the other gradients keep their bits."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=12, log_scale_range=(0.003, 0.05))
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    w, u = (torch.from_numpy(x).to(cuda) for x in _weights(hw, 2))
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True,
                                              render_depth=True)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    _, pg = pipeline.render_view_backward(P, st, d, clamped_img=img, d_depth=u)
    on, cam_on = _project(cuda, P, st, pg, True)
    off, cam_off = _project(cuda, P, st, pg, False)
    assert torch.equal(cam_on[1], cam_off[1])
    keep = [0, 1, 3]
    assert torch.equal(cam_on[0][:, keep], cam_off[0][:, keep])
    for a, b in zip(on[1:], off[1:]):
        assert torch.equal(a, b)
    # the column-2 difference is the depth term: sum_i p~_ik dz_i over the visible Gaussians
    S = P["xyz"].shape[-1]
    ids = st.chunk_ids[: st.n_chunks_visible]
    p = P["xyz"].index_select(1, ids).reshape(3, -1).double()
    dz = pg[0, : st.n_chunks_visible * S, 10].double()
    want = torch.cat([p @ dz, dz.sum()[None]])
    got = (cam_on[0][:, 2] - cam_off[0][:, 2]).double()
    assert dz.abs().max() > 0
    assert (got - want).abs().max() <= 1e-4 * want.abs().max(), (got, want)


def test_workspace_depth_gradient_padding_and_forward_check(cuda, deterministic):
    """ViewWorkspace.backward: an [H,W] d_depth after a padded one with non-zero padding gives the same gradients as on a fresh
    workspace (the stale padding is cleared), and a d_depth after a forward without depth is refused."""
    hw, tile = (90, 120), (8, 16)           # neither side a multiple of the tile: the planes have padding
    P, A, cams, w, u = _setup_views(cuda, hw=hw)
    Hp, Wp = 96, 128
    u = u[..., :hw[0], :hw[1]]
    big = torch.ones((1, 1, Hp, Wp), device=cuda) * 7.0
    big[..., :hw[0], :hw[1]] = u

    def run(ws, grads):
        acc = GradAccumulator(P)
        for g in grads:
            acc.zero_()
            ws.forward(P, A[0], A[1], cams[0], 3, render_depth=True)
            ws.backward(P, w[..., :hw[0], :hw[1]], 3, acc.grads(), d_depth=g)
        torch.cuda.synchronize()
        return {k: v.clone() for k, v in acc.grads().items()}

    mk = lambda: pipeline.ViewWorkspace(P, hw, tile, 1 << 20, 32, use_graphs=False)
    fresh = run(mk(), [u])
    stale = run(mk(), [big, u])
    for k in PARAM_KEYS:
        assert torch.equal(fresh[k], stale[k]), k
    ws = mk()
    acc = GradAccumulator(P)
    ws.forward(P, A[0], A[1], cams[0], 3, render_depth=True)
    ws.forward(P, A[0], A[1], cams[1], 3)
    with pytest.raises(RuntimeError, match="did not render depth"):
        ws.backward(P, w[..., :hw[0], :hw[1]], 3, acc.grads(), d_depth=u)


def test_c2_one_view_matches_restatement(cuda):
    """One full-size view (1M Gaussians, 1920x1080, SH degree 3, 8x16 tiles) with a colour and a depth loss against the
    restatement: D, the image, the six gradients and the camera gradient."""
    H, W, tile, deg = 1080, 1920, (8, 16), 3
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0)
    params = {k: p[k] for k in PARAM_KEYS}
    aabb = (p["cluster_origin"], p["cluster_extend"])
    cam = scene.make_camera(0, 64, W, H)
    g = np.random.default_rng(7)
    w, u = g.normal(size=(1, 3, H, W)).astype(np.float32), g.normal(size=(1, 1, H, W)).astype(np.float32)
    o0 = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, render_depth=True)
    frag = o0["fragile"][:, :H, :W].copy()
    assert frag.mean() < 0.10
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, (H, W), tile, clamp_zero=True,
                                              render_depth=True)
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
    ok = ~frag[:, None]
    errs = {"img": np.abs(img.cpu().numpy()[..., :H, :W] - o0["img"])[np.broadcast_to(ok, o0["img"].shape)].max(),
            "D": np.abs(st.depth.cpu().numpy()[..., :H, :W] - o0["depth"])[ok].max() / np.abs(o0["depth"]).max()}
    w, u = w * ok, u * ok
    ref = fo.render_forward_backward(params, aabb, cam, (H, W), tile, deg, lambda img: w, render_depth=True,
                                     d_depth_fn=lambda D_, T_: (u, None))
    ref64 = as_f64(ref)
    d_view, d_proj = fo.camera_backward(params, ref64, cam, (H, W), sh_degree=deg)
    d = torch.zeros_like(img)
    d[..., :H, :W] = torch.from_numpy(w).to(cuda)
    cg = torch.empty((2, 4, 4), device=cuda)
    grads, _ = pipeline.render_view_backward(P, st, d, clamped_img=img, camera_grad=cg, d_depth=torch.from_numpy(u).to(cuda))
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k, gr in zip(PARAM_KEYS, grads):
        errs[k] = scaled_err(gr.cpu().numpy()[..., :nvis, :], ref["grads"][k][..., :nvis, :])
    errs["d_view"] = np.abs(cg[0].cpu().numpy() - d_view).max() / np.abs(d_view).max()
    errs["d_proj"] = np.abs(cg[1].cpu().numpy() - d_proj).max() / np.abs(d_proj).max()
    print(f"C2 depth view ({frag.mean() * 100:.2f} % fragile): " + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    assert errs.pop("img") < 1e-4
    for k, e in errs.items():
        assert e < 2e-4, (k, e)


def test_train_colmap_depth_weight_lowers_the_expected_depth_error(cuda, tmp_path):
    """examples/train_colmap.py --depth-weight on a small synthetic dataset (make_dataset writes the hidden scene's expected depth):
    the GPU-driven path trains with the term, and the expected-depth error ends lower than in the same run without it."""
    import importlib.util
    import os
    spec = importlib.util.spec_from_file_location("train_colmap", os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples",
                                                                              "train_colmap.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    root = mod.make_dataset(str(tmp_path / "ds"), n_gaussians=8000, n_views=8, hw=(96, 160), n_points=4000, dev=cuda)
    assert len(os.listdir(os.path.join(root, "depths"))) == 8
    res = {}
    for wd in (0.0, 0.3):
        m = {}
        hist, psnr = mod.train(root, iters=120, views_per_step=4, log=lambda *_: None, depth_weight=wd, metrics=m)
        res[wd] = (hist, psnr, m["ed_error"])
    print("train_colmap: " + ", ".join(f"depth weight {k}: loss {v[0][0]:.4f} -> {v[0][-1]:.4f}, PSNR {v[1]:.2f} dB, ED error {v[2]:.4f}"
                                       for k, v in res.items()))
    assert res[0.3][0][-1] < res[0.3][0][0]
    assert res[0.3][2] < res[0.0][2]
