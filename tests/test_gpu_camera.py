"""Learnable cameras on the GPU: create_viewproj against the CPU restatement and the reference's fixture; the camera gradient of
render_view (d view_matrix, d proj_matrix) against the oracle, its translation identity at 1M Gaussians, its determinism and its
agreement across the synchronising, autograd and graph-replayed paths; autograd through CreateViewProj; pose recovery."""
import os

import numpy as np
import pytest
import torch

from litegs_b200 import fused, pipeline, render, scene, wrapper
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import camera_oracle as co
from tests.util import PARAM_KEYS, ZF, ZN, as_f64, deterministic, oracle_case, rot_err_deg, to_torch, view_params

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "viewproj.npz")


def test_create_viewproj_matches_oracle_and_reference(cuda):
    g = np.load(GOLD)
    H, W = 1080, 1920
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    got = [a.cpu().numpy() for a in fused.create_viewproj_forward(T(g["view_params"]), T(g["recp"]), H, W, ZN, ZF)]
    want = co.create_viewproj_forward(g["view_params"].astype(np.float64), g["recp"].astype(np.float64), H, W, ZN, ZF)
    for k, a, b in zip(("view", "proj", "viewproj", "frustumplane"), got, want):
        assert np.abs(a - g[k]).max() <= 1e-5 * np.abs(g[k]).max(), k
        assert np.abs(a - b).max() <= 1e-5 * np.abs(b).max(), k
    gp, gr = fused.create_viewproj_backward(T(g["g_view"]), T(g["g_proj"]), T(g["g_viewproj"]), T(g["view_params"]), T(g["recp"]), H, W, ZN, ZF)
    wp, wr = co.create_viewproj_backward(g["g_view"], g["g_proj"], g["g_viewproj"], g["view_params"].astype(np.float64),
                                         g["recp"].astype(np.float64), H, W, ZN, ZF)
    gp = gp.cpu().numpy()
    assert np.abs(gp - g["grad_view_params"]).max() <= 1e-5 * np.abs(g["grad_view_params"]).max()
    assert np.abs(gp - wp).max() <= 1e-5 * np.abs(wp).max()
    assert abs(float(gr[0]) - wr[0]) <= 1e-5 * max(1.0, abs(wr[0]))            # deterministic sum over the 5 views
    _, gr1 = fused.create_viewproj_backward(T(g["g_view"][:1]), T(g["g_proj"][:1]), T(g["g_viewproj"][:1]), T(g["view_params"][:1]), T(g["recp"]),
                                            H, W, ZN, ZF)
    assert abs(float(gr1[0]) - float(g["grad_recp_v1"][0])) <= 1e-5 * max(1.0, abs(float(g["grad_recp_v1"][0])))


def _camera_grad_direct(P, A, C, deg, hw, tile, w, accumulate_into=None):
    """pipeline forward + backward of one view with the camera gradient on -> (camera_grad [2,4,4], compacted grads or None)."""
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], deg, hw, tile, clamp_zero=True)
    d = torch.zeros_like(img)
    d[..., :hw[0], :hw[1]] = w
    cg = torch.empty((2, 4, 4), dtype=torch.float32, device=img.device)
    grads, _ = pipeline.render_view_backward(P, st, d, accumulate_into=accumulate_into, clamped_img=img, camera_grad=cg)
    return cg, grads, st


@pytest.mark.parametrize("deg,tile,view", [(3, (16, 16), 0), (3, (8, 16), 3), (0, (8, 16), 5), (0, (16, 16), 6)])
def test_render_view_camera_gradient_matches_oracle(cuda, deterministic, deg, tile, view):
    hw = (96, 128)
    params, aabb, cam, w, frag, ref = oracle_case(4000, hw, tile, deg, seed=11, view=view)
    d_view, d_proj, _ = co.camera_backward(params, as_f64(ref), cam, hw)
    P, A, C = to_torch(params, aabb, cam, cuda, grad=False)
    V = C["view"].clone().requires_grad_(True)
    Pm = C["proj"].clone().requires_grad_(True)
    pp = PipelineParams(tile_size=tile)
    img = render.render_view(A[0], A[1], C["frustumplane"], V, Pm, P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"],
                             deg, hw, pp)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    gv, gp = V.grad.cpu().numpy()[0], Pm.grad.cpu().numpy()[0]
    ev = np.abs(gv - d_view).max() / np.abs(d_view).max()
    ep = np.abs(gp - d_proj).max() / np.abs(d_proj).max()
    print(f"camera gradient vs oracle (deg {deg}, tile {tile}, view {view}): d_view {ev:.2e}, d_proj {ep:.2e} of their maximum")
    assert ev < 1e-4 and ep < 1e-4
    # the direct entry point gives the same bits as the autograd Function
    cg, _, _ = _camera_grad_direct(P, A, C, deg, hw, tile, torch.from_numpy(w).to(cuda))
    assert np.array_equal(cg[0].cpu().numpy(), gv) and np.array_equal(cg[1].cpu().numpy(), gp)


def test_translation_identity_and_determinism_at_1m(cuda, deterministic):
    """C2 (1M Gaussians, 1920x1080, 8x16 tiles): sum_i d xyz_i = V3x3 . d_view[3,:3] within fp32 summation error; with the
    camera gradient on, the six parameter gradients are bit-identical to a run with it off; two runs give the same bits."""
    H, W = 1080, 1920
    hw, tile = (H, W), (8, 16)
    p = scene.make_scene(1_000_000, sh_degree=3, seed=0, log_scale_range=(0.002, 0.02))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(3, 64, W, H).items()}
    w = torch.randn((1, 3, H, W), generator=torch.Generator(device="cpu").manual_seed(4)).to(cuda)
    acc = GradAccumulator(P)
    acc.zero_()
    cg, _, _ = _camera_grad_direct(P, A, C, 3, hw, tile, w, accumulate_into=acc.grads())
    gx = acc.grads()["xyz"].double().reshape(3, -1)
    s = gx.sum(dim=1).cpu().numpy()
    mag = gx.abs().sum(dim=1).cpu().numpy()
    rhs = C["view"][0, :3, :3].double().cpu().numpy() @ cg[0, 3, :3].double().cpu().numpy()
    err = np.abs(s - rhs) / mag
    print(f"C2 translation identity: sum d xyz {s}, V3x3 . d_view[3,:3] {rhs}, error / sum|d xyz| {err}")
    assert np.all(err < 1e-5)
    on = {k: v.clone() for k, v in acc.grads().items()}
    acc.zero_()
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True)
    d = torch.zeros_like(img)
    d[..., :H, :W] = w
    pipeline.render_view_backward(P, st, d, accumulate_into=acc.grads(), clamped_img=img)
    for k in PARAM_KEYS:
        assert torch.equal(acc.grads()[k], on[k]), k
    cg2, grads, _ = _camera_grad_direct(P, A, C, 3, hw, tile, w)
    assert torch.equal(cg, cg2)


def _setup_views(cuda, n=8000, hw=(72, 96), seed=6):
    p = scene.make_scene(n, sh_degree=3, cube=1.5, seed=seed, log_scale_range=(0.02, 0.08))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    return P, A, cams, w


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
    return cg.clone()


@pytest.mark.parametrize("n_streams", [1, 3])
def test_render_views_camera_grads_on_every_path(cuda, deterministic, n_streams):
    """Slot i of camera_grads is view i's camera gradient: per-view render_view runs, the direct synchronising path, the autograd
    path and the GPU-driven workspaces (eager, captured and replayed, with other cameras in between) agree bit for bit."""
    hw, tile = (72, 96), (8, 16)
    P, A, cams, w = _setup_views(cuda, hw=hw)
    pp = PipelineParams(tile_size=tile)
    acc = GradAccumulator(P)
    va, vb = [0, 1, 2, 3, 4, 5], [6, 7, 8, 9, 10, 11]
    # per view, one render_view each
    per_view = {}
    for v in va + vb:
        cg, _, _ = _camera_grad_direct(P, A, cams[v], 3, hw, tile, w * (1.0 + 0.1 * v))
        per_view[v] = cg
    ref = {tuple(va): torch.stack([per_view[v] for v in va]), tuple(vb): torch.stack([per_view[v] for v in vb])}
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    try:
        pipeline.SYNC_FREE = False
        assert torch.equal(_views_batch(P, A, cams, w, hw, pp, acc, va, n_streams), ref[tuple(va)])
        assert torch.equal(_views_batch(P, A, cams, w, hw, pp, acc, vb, n_streams, direct=False), ref[tuple(vb)])
        pipeline.SYNC_FREE = True
        # batch 1 measures the capacities, 2 runs eagerly on the workspaces, 3 captures the graphs, 4.. replay them
        for views in (va, va, vb, va, vb, va):
            assert torch.equal(_views_batch(P, A, cams, w, hw, pp, acc, views, n_streams), ref[tuple(views)]), views
        render.check_views(wait=True)
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


def test_workspace_replay_equals_synchronising_path(cuda, deterministic):
    """A ViewWorkspace with graph capture: the camera gradient of every replay equals the synchronising path's, bit for bit, and
    a replay picks up a new camera.  Turning the camera gradient off and on changes the graph signature, not the results."""
    hw, tile = (70, 100), (8, 16)
    P, A, cams, w = _setup_views(cuda, hw=hw)
    pairs, bits = pipeline.probe_view_sizes(P, A[0], A[1], cams, 3, hw, tile)
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=int(pairs * 1.3), planned_depth_bits=32, use_graphs=True)
    acc = GradAccumulator(P)
    side = torch.cuda.Stream(device=cuda)                  # graphs are not captured on the legacy default stream
    with torch.cuda.stream(side):
        for rnd in range(3):
            for v in (0, 4, 9):
                want, _, _ = _camera_grad_direct(P, A, cams[v], 3, hw, tile, w)
                ws.forward(P, A[0], A[1], cams[v], 3)
                got = torch.full((2, 4, 4), float("nan"), device=cuda)
                ws.backward(P, w, 3, acc.grads(), camera_grad=got)
                side.synchronize()
                assert torch.equal(got, want), (rnd, v)
                if rnd == 1:                                    # an off run in between: its own graph, no camera output
                    ws.forward(P, A[0], A[1], cams[v], 3)
                    ws.backward(P, w, 3, acc.grads())
    assert any(k[0] == "bwd" and k[1][-1] for k in ws._graphs) and any(k[0] == "bwd" and not k[1][-1] for k in ws._graphs)


def test_autograd_through_create_viewproj(cuda, deterministic):
    """CreateViewProj.apply -> render_view -> backward fills extr.grad with create_viewproj_backward of the direct d_view/d_proj."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam, w, frag, ref = oracle_case(4000, hw, tile, 3, seed=12, view=2)
    P, A, _ = to_torch(params, aabb, cam, cuda, grad=False)
    extr = torch.tensor(np.stack([view_params(cam)]), dtype=torch.float32, device=cuda).requires_grad_(True)
    intr = torch.tensor([float(cam["proj"][0, 0, 0])], dtype=torch.float32, device=cuda).requires_grad_(True)
    pp = PipelineParams(tile_size=tile)
    view, proj, _, planes = wrapper.CreateViewProj.apply(extr, intr, hw[0], hw[1], ZN, ZF)
    wt = torch.from_numpy(w).to(cuda)
    img = render.render_view(A[0], A[1], planes, view, proj, P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, hw, pp)[0]
    (img * wt).sum().backward()
    Cd = dict(view=view.detach(), proj=proj.detach(), frustumplane=planes)
    cg, _, _ = _camera_grad_direct(P, A, Cd, 3, hw, tile, wt)
    z = torch.zeros((1, 4, 4), device=cuda)
    want, want_r = fused.create_viewproj_backward(cg[0:1], cg[1:2], z, extr.detach(), intr.detach(), hw[0], hw[1], ZN, ZF)
    assert torch.equal(extr.grad, want) and torch.equal(intr.grad, want_r)
    assert float(extr.grad.abs().max()) > 0


def test_pose_recovery(cuda):
    """Gaussians at ground truth, 4 cameras perturbed by 1 degree of rotation and 2 % of their distance in translation; Adam on the
    extrinsics alone with an L1 loss brings every camera's rotation and translation errors below 25 % of their initial values."""
    hw, tile = (120, 160), (8, 16)
    H, W = hw
    p = scene.make_scene(20_000, sh_degree=3, seed=8, log_scale_range=(0.03, 0.1))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    n = 4
    true = np.stack([view_params(scene.make_camera(v, n, W, H)) for v in range(n)])
    recp = torch.tensor([float(scene.make_camera(0, n, W, H)["proj"][0, 0, 0])], device=cuda)
    pp = PipelineParams(tile_size=tile)
    rng = np.random.default_rng(1)
    noisy = true.copy()
    for v in range(n):
        axis = rng.normal(size=3); axis /= np.linalg.norm(axis)
        a = np.radians(1.0)
        dq = np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * axis])
        r1, v1 = true[v, 0], true[v, 1:4]
        r2, v2 = dq[0], dq[1:]
        noisy[v, :4] = np.concatenate([[r1 * r2 - v1 @ v2], r1 * v2 + r2 * v1 + np.cross(v1, v2)])
        d = rng.normal(size=3); d /= np.linalg.norm(d)
        noisy[v, 4:] = true[v, 4:] + 0.02 * np.linalg.norm(true[v, 4:]) * d
    with torch.no_grad():
        tv, tp, _, tpl = fused.create_viewproj_forward(torch.tensor(true, dtype=torch.float32, device=cuda), recp, H, W, ZN, ZF)
        gts = [render.render_view(A[0], A[1], tpl[v:v + 1], tv[v:v + 1], tp[v:v + 1], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                                  P["opacity"], 3, hw, pp)[0] for v in range(n)]
    extr = torch.tensor(noisy, dtype=torch.float32, device=cuda).requires_grad_(True)
    rot0 = [rot_err_deg(noisy[v], true[v]) for v in range(n)]
    tr0 = [float(np.linalg.norm(noisy[v, 4:] - true[v, 4:])) for v in range(n)]
    steps = 300
    opt = torch.optim.Adam([extr], lr=3e-3)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda s: 0.01 ** (s / steps))
    for _ in range(steps):
        view, proj, _, planes = wrapper.CreateViewProj.apply(extr, recp, H, W, ZN, ZF)
        loss = 0.0
        for v in range(n):
            img = render.render_view(A[0], A[1], planes[v:v + 1].detach(), view[v:v + 1], proj[v:v + 1], P["xyz"], P["scale"], P["rot"],
                                     P["sh_0"], P["sh_rest"], P["opacity"], 3, hw, pp)[0]
            loss = loss + (img - gts[v]).abs().mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        sched.step()
    est = extr.detach().double().cpu().numpy()
    rot1 = [rot_err_deg(est[v], true[v]) for v in range(n)]
    tr1 = [float(np.linalg.norm(est[v, 4:] - true[v, 4:])) for v in range(n)]
    print("pose recovery: rotation error (deg)", [f"{a:.3f} -> {b:.4f}" for a, b in zip(rot0, rot1)],
          "translation error", [f"{a:.4f} -> {b:.5f}" for a, b in zip(tr0, tr1)])
    for v in range(n):
        assert rot1[v] < 0.25 * rot0[v] and tr1[v] < 0.25 * tr0[v], (v, rot0[v], rot1[v], tr0[v], tr1[v])

