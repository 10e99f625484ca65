"""Depth-normal consistency on the GPU (csrc/geometry.cu through litegs_b200.geometry): the kernel against the fp32 numpy
restatement (tests/depth_normal_oracle.py) on random and rendered inputs at three sizes; bit-reproducibility, strided inputs and
CUDA-graph replay; render_views' direct, autograd and graph-replayed paths with the term switched on and off; rotations of flat
Gaussians on a plane turned toward the plane by the term alone; examples/train_colmap.py --depth-normal-weight without depth or
normal targets."""
import importlib.util
import os
import shutil

import numpy as np
import pytest
import torch

from litegs_b200 import geometry, pipeline, render, scene
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import depth_normal_oracle as dn
from tests.util import PARAM_KEYS, deterministic, scaled_err  # noqa: F401  (deterministic is a fixture)

pytestmark = pytest.mark.gpu

SIZES = [(37, 53), (64, 128), (1080, 1920)]       # odd; a multiple of the 16 x 64 CTA tile; full HD


def _random_inputs(hw, seed):
    """A bumpy depth field, alpha in (0.3, 1) (about a quarter of the pixels at or below alpha_min = 0.5), random normals with a
    few zero pixels -> numpy D, T [1,1,H,W], N [1,3,H,W], proj [1,4,4]."""
    H, W = hw
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    ed = 4.0 + np.sin(0.05 * x) * np.cos(0.07 * y) + 0.02 * rng.normal(size=(H, W))
    alpha = rng.uniform(0.3, 1.0, (H, W))
    N = rng.normal(size=(3, H, W)) * rng.uniform(0.0, 1.0, (1, H, W))
    N[:, rng.random((H, W)) < 0.01] = 0.0
    P = dn.proj_matrix(0.9 * W, 0.9 * W, H, W)
    return ((alpha * ed)[None, None].astype(np.float32), (1 - alpha)[None, None].astype(np.float32), N[None].astype(np.float32), P)


def _rendered_inputs(cuda, hw, seed=0):
    """D, T, N of a rendered scene (depth and normals on), as the strided [..., :H, :W] views of the padded planes, and proj."""
    H, W = hw
    p = scene.make_scene(20000, sh_degree=3, seed=seed, log_scale_range=(0.01, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    C = {k: torch.from_numpy(v).to(cuda) for k, v in scene.make_camera(2, 8, W, H, radius=2.2).items()}
    _, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, (8, 16), clamp_zero=True,
                                            render_depth=True, render_normal=True)
    return st.depth[..., :H, :W], st.T[..., :H, :W], st.normal[..., :H, :W], C["proj"]


@pytest.mark.parametrize("source", ["random", "rendered"])
@pytest.mark.parametrize("hw", SIZES)
def test_kernel_matches_restatement(cuda, hw, source):
    """The n_d mask is identical; n_d within 1e-5, the loss within 1e-5 relative and the three gradients within 1e-4 of their
    maximum of the fp32 restatement."""
    if source == "random":
        Dn, Tn, Nn, Pn = _random_inputs(hw, hw[0])
        D, T, N, Pt = (torch.from_numpy(x).to(cuda) for x in (Dn, Tn, Nn, Pn))
    else:
        D, T, N, Pt = _rendered_inputs(cuda, hw)
        Dn, Tn, Nn, Pn = (x.cpu().numpy() for x in (D, T, N, Pt))
    w, up = 0.3, 1.7
    ref = dn.forward_backward(Dn, Tn, Nn, Pn, weight=w, upstream=up, dtype=np.float32)
    nd, mask = geometry.depth_normal(D, T, Pt)
    loss, gD, gT, gN = geometry.depth_normal_loss_and_grad(D, T, N, Pt, w, upstream=up)
    m = mask[0, 0].cpu().numpy()
    errs = {"n_d": float(np.abs(nd[0].cpu().numpy() - ref["nd"]).max()),
            "loss": abs(float(loss) - ref["loss"]) / abs(ref["loss"]),
            "d_depth": scaled_err(gD[0, 0].cpu().numpy(), ref["dD"]), "d_trans": scaled_err(gT[0, 0].cpu().numpy(), ref["dT"]),
            "d_normal": scaled_err(gN[0].cpu().numpy(), ref["dN"])}
    print(f"depth-normal {source} {hw}: mask on {100 * m.mean():.1f} % of the pixels, loss {float(loss):.6e}; "
          + ", ".join(f"{k} {e:.1e}" for k, e in errs.items()))
    assert m.mean() > 0.1
    assert np.array_equal(m, ref["mask"]), int((m != ref["mask"]).sum())
    assert errs.pop("n_d") < 1e-5
    assert errs.pop("loss") < 1e-5
    for k, e in errs.items():
        assert e < 1e-4, (k, e)


def test_small_sizes_and_refusals(cuda):
    """Sizes without an interior pixel give a zero loss and zero gradients; bad inputs are refused at the boundary."""
    for hw in ((1, 1), (2, 50), (50, 2)):
        D, T, N, P = (torch.from_numpy(x).to(cuda) for x in _random_inputs(hw, 1))
        loss, gD, gT, gN = geometry.depth_normal_loss_and_grad(D, T, N, P, 1.0)
        assert float(loss) == 0 and not gD.any() and not gT.any() and not gN.any()
        assert not geometry.depth_normal(D, T, P)[0].any()
    D, T, N, P = (torch.from_numpy(x).to(cuda) for x in _random_inputs((20, 30), 2))
    with pytest.raises(RuntimeError, match="float32 CUDA"):
        geometry.depth_normal_loss_and_grad(D.cpu(), T, N, P, 1.0)
    with pytest.raises(RuntimeError, match=r"\[1,3,20,30\]"):
        geometry.depth_normal_loss_and_grad(D, T, N[:, :2], P, 1.0)
    with pytest.raises(RuntimeError, match="alpha_min"):
        geometry.depth_normal(D, T, P, alpha_min=-0.1)
    with pytest.raises(RuntimeError, match="proj"):
        geometry.depth_normal(D, T, P[0, :3])
    with pytest.raises(RuntimeError, match="enable_transmitance"):
        geometry.depth_normal_loss(D, None, N, P, 1.0)
    with pytest.raises(RuntimeError, match="render_normal"):
        geometry.depth_normal_loss(D, T, None, P, 1.0)


def test_deterministic_strided_and_graph_replay(cuda):
    """Two calls give the same bits; [..., :H, :W] views of padded planes give the bits of their contiguous copies; the call
    captured in a CUDA graph replays to the same bits."""
    hw = (270, 330)
    D, T, N, P = (torch.from_numpy(x).to(cuda) for x in _random_inputs(hw, 3))
    a = geometry.depth_normal_loss_and_grad(D, T, N, P, 0.5)
    b = geometry.depth_normal_loss_and_grad(D, T, N, P, 0.5)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert torch.equal(geometry.depth_normal(D, T, P)[0], geometry.depth_normal(D, T, P)[0])
    pads = [torch.full((1, x.shape[1], hw[0] + 6, hw[1] + 10), 1e3, device=cuda) for x in (D, T, N)]
    for pd, x in zip(pads, (D, T, N)):
        pd[..., :hw[0], :hw[1]] = x
    views = [pd[..., :hw[0], :hw[1]] for pd in pads]
    assert not views[0].is_contiguous()
    c = geometry.depth_normal_loss_and_grad(*views, P, 0.5)
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    assert torch.equal(geometry.depth_normal(views[0], views[1], P)[0], geometry.depth_normal(D, T, P)[0])
    s = torch.cuda.Stream(cuda)
    s.wait_stream(torch.cuda.current_stream(cuda))
    with torch.cuda.stream(s):
        geometry.depth_normal_loss_and_grad(*views, P, 0.5)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            out = geometry.depth_normal_loss_and_grad(*views, P, 0.5)
    torch.cuda.current_stream(cuda).wait_stream(s)
    for x in out:
        x.fill_(float("nan"))
    g.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(a, out))


def test_render_views_paths_agree(cuda, deterministic):  # noqa: F811
    """A colour loss plus the consistency term: the direct path (loss_and_grad_fn), the autograd paths (loss_fn through
    depth_normal_loss, with and without render_view's autograd Function) and the graph-replayed workspace path give the same
    parameter and camera gradients bit for bit, with the term switched on and off between batches."""
    hw, tile = (72, 96), (8, 16)
    p = scene.make_scene(8000, sh_degree=3, cube=1.5, seed=6, log_scale_range=(0.005, 0.05))
    P = {k: torch.from_numpy(p[k]).to(cuda) for k in PARAM_KEYS}
    A = [torch.from_numpy(p[k]).to(cuda) for k in ("cluster_origin", "cluster_extend")]
    cams = [{k: torch.from_numpy(x).to(cuda) for k, x in scene.make_camera(v, 12, hw[1], hw[0]).items()} for v in range(12)]
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    views, weight = [0, 1, 2, 3, 4, 5], 20.0
    pp_on = PipelineParams(tile_size=tile, render_depth=True, render_normal=True)
    pp_off = PipelineParams(tile_size=tile)
    proj = lambda i: cams[views[i]]["proj"]
    fns = {
        ("grad", True): lambda i, img, depth, trans, normal: (
            lambda t: ((img * w).sum() + t[0], w, *t[1:]))(geometry.depth_normal_loss_and_grad(depth, trans, normal, proj(i), weight)),
        ("grad", False): lambda i, img: ((img * w).sum(), w),
        ("autograd", True): lambda i, img, depth, trans, normal: (img * w).sum() + geometry.depth_normal_loss(depth, trans, normal, proj(i),
                                                                                                               weight),
        ("autograd", False): lambda i, img: (img * w).sum(),
    }
    acc = GradAccumulator(P)

    def batch(on, form, direct=True):
        acc.zero_()
        cg = torch.full((len(views), 2, 4, 4), float("nan"), device=cuda)
        keep = render._DIRECT_VIEWS
        try:
            render._DIRECT_VIEWS = direct
            fn = fns[(form, on)]
            render.render_views(len(views), lambda i: cams[views[i]], fn if form == "autograd" else None, A[0], A[1], P["xyz"], P["scale"],
                                P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 3, hw, pp_on if on else pp_off, acc.grads(), n_streams=3,
                                camera_grads=cg, loss_and_grad_fn=fn if form == "grad" else None)
        finally:
            render._DIRECT_VIEWS = keep
        torch.cuda.synchronize()
        return cg.clone(), {k: v.clone() for k, v in acc.grads().items()}

    same = lambda a, b: torch.equal(a[0], b[0]) and all(torch.equal(a[1][k], b[1][k]) for k in PARAM_KEYS)
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    try:
        pipeline.SYNC_FREE = False
        want = {on: batch(on, "grad") for on in (True, False)}
        assert not torch.equal(want[True][1]["rot"], want[False][1]["rot"])
        assert not torch.equal(want[True][0], want[False][0])
        assert same(batch(True, "autograd"), want[True])
        assert same(batch(True, "autograd", direct=False), want[True])
        pipeline.SYNC_FREE = True
        for on in (True, False, True, True, False, True):
            assert same(batch(on, "grad"), want[on]), on
        assert same(batch(True, "autograd"), want[True])
        render.check_views(wait=True)
        ws = next(iter(render._slot_cache.values())).ws[0]
        assert any(k[0] == "bwd" for k in ws._graphs)
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()


def _plane_scene(n=6144, seed=0):
    """Flat Gaussians (one log-scale far smaller) with random rotations, centred on a tilted plane through the origin, seen by a
    camera at distance 3 -> (params on the CPU, plane's world normal)."""
    rng = np.random.default_rng(seed)
    uv = rng.uniform(-1.3, 1.3, (2, n))
    tilt = np.array([0.35, -0.25])
    xyz = np.stack([uv[0], uv[1], tilt[0] * uv[0] + tilt[1] * uv[1]])
    nrm = np.array([-tilt[0], -tilt[1], 1.0])
    nrm /= np.linalg.norm(nrm)
    order = scene.morton_order(xyz)
    xyz = xyz[:, order]
    q = rng.normal(size=(4, n))
    q /= np.linalg.norm(q, axis=0)
    scale = np.log(np.array([0.05, 0.05, 0.004]))[:, None] * np.ones((1, n))
    scale = np.take_along_axis(scale, np.argsort(rng.random((3, n)), axis=0), axis=0)       # the thin axis in a random slot
    C = 128
    cl = lambda a: scene.cluster(a.astype(np.float32), C)
    params = dict(xyz=cl(xyz), scale=cl(scale), rot=cl(q), sh_0=cl(np.full((1, 3, n), 0.8)), sh_rest=np.zeros((15, 3, n // C, C), np.float32),
                  opacity=cl(np.full((1, n), 2.5)))
    origin, extend = scene.cluster_aabb(params["xyz"], params["scale"], params["rot"])
    return params, (origin, extend), nrm


def test_term_turns_flat_gaussians_toward_the_plane(cuda):
    """Optimising only the rotations with Adam on the consistency term alone: the mean angle between N / |N| and the plane's normal
    over the covered pixels falls below half its initial value."""
    hw = (160, 160)
    params, aabb, nrm_w = _plane_scene()
    V = scene.look_at_view_matrix(np.array([0.4, -0.3, -3.0]))
    Pm = scene.proj_matrix(hw[1], hw[0], 50.0)
    cam = dict(view=V[None].astype(np.float32), proj=Pm[None].astype(np.float32), frustumplane=scene.frustum_planes(V, Pm)[None])
    n_view = nrm_w @ V[:3, :3]
    n_view = n_view if n_view @ (np.array([0.0, 0.0, 0.0, 1.0]) @ V)[:3] < 0 else -n_view       # camera-facing, at the origin
    P = {k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in params.items()}
    A = [torch.from_numpy(a).to(cuda) for a in aabb]
    C = {k: torch.from_numpy(np.ascontiguousarray(v)).to(cuda) for k, v in cam.items()}
    P["rot"].requires_grad_(True)
    pp = PipelineParams(tile_size=(8, 16), cluster_size=128, sparse_grad=False, enable_transmitance=True, render_depth=True,
                        render_normal=True)
    opt = torch.optim.Adam([P["rot"]], lr=0.02)
    target = torch.tensor(n_view, dtype=torch.float32, device=cuda).view(1, 3, 1, 1)

    def angle(normal, trans):
        cov = (1 - trans) > 0.5
        u = normal / normal.norm(dim=1, keepdim=True).clamp_min(1e-12)
        return float(torch.rad2deg(torch.arccos((u * target).sum(1, keepdim=True).clamp(-1, 1)))[cov].mean())

    angles = []
    for it in range(150):
        opt.zero_grad()
        img, trans, depth, normal, _ = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"],
                                                          P["sh_0"], P["sh_rest"], P["opacity"], 0, hw, pp)
        if it == 0:
            nd, mask = geometry.depth_normal(depth, trans, C["proj"])
            err = float(torch.rad2deg(torch.arccos((nd * target).sum(1, keepdim=True).clamp(-1, 1)))[mask].mean())
            cover = float(mask.float().mean())
            assert cover > 0.3, cover
        angles.append(angle(normal.detach(), trans.detach()))
        loss = geometry.depth_normal_loss(depth, trans, normal, C["proj"], 1.0)
        loss.backward()
        opt.step()
    print(f"flat Gaussians on a plane, rotations trained on the consistency term alone: mean angle to the plane normal "
          f"{angles[0]:.2f} -> {angles[-1]:.2f} degrees (n_d defined on {100 * cover:.1f} % of the pixels, {err:.2f} degrees from it)")
    assert angles[-1] < 0.5 * angles[0]


def _train_colmap():
    spec = importlib.util.spec_from_file_location("train_colmap", os.path.join(os.path.dirname(os.path.dirname(__file__)), "examples",
                                                                              "train_colmap.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_train_colmap_depth_normal_weight(cuda, tmp_path):
    """--depth-normal-weight 0.1 trains on a dataset without depths/ and normals/ and its loss falls; reported, not gated: the
    consistency angle, and the angle to the hidden scene's normals with and without the term (the synthetic scene is a volume,
    not a surface)."""
    mod = _train_colmap()
    root = mod.make_dataset(str(tmp_path / "ds"), n_gaussians=8000, n_views=8, hw=(96, 160), n_points=4000, dev=cuda)
    shutil.move(os.path.join(root, "normals"), str(tmp_path / "hidden_normals"))
    shutil.rmtree(os.path.join(root, "depths"))
    m = {}
    hist, psnr = mod.train(root, iters=120, views_per_step=4, log=lambda *_: None, depth_normal_weight=0.1, metrics=m)
    assert hist[-1] < hist[0]
    assert "depth_normal_angle" in m and "normal_angle" not in m
    # the same runs with the hidden normals back in place, as an evaluation target only (no normal loss)
    shutil.move(str(tmp_path / "hidden_normals"), os.path.join(root, "normals"))
    res = {}
    for wdn in (0.0, 0.1):
        mm = {}
        h, ps = mod.train(root, iters=120, views_per_step=4, log=lambda *_: None, depth_normal_weight=wdn, metrics=mm)
        res[wdn] = (h, ps, mm)
    print(f"train_colmap --depth-normal-weight 0.1 without targets: loss {hist[0]:.4f} -> {hist[-1]:.4f}, PSNR {psnr:.2f} dB, "
          f"consistency angle {m['depth_normal_angle']:.2f} deg; angle to the hidden normals without the term "
          f"{res[0.0][2]['normal_angle']:.2f} deg (PSNR {res[0.0][1]:.2f} dB), with it {res[0.1][2]['normal_angle']:.2f} deg "
          f"(consistency {res[0.1][2]['depth_normal_angle']:.2f} deg, PSNR {res[0.1][1]:.2f} dB)")
    assert res[0.1][0][-1] < res[0.1][0][0]
