"""The drop-in, exercised (VERDICT "What's weak" 2): the reference's OWN, UNMODIFIED Python -- ``litegs/utils/wrapper.py``,
``litegs/render/__init__.py``, ``litegs/utils/statistic_helper.py``, ``litegs/training/trainer.py`` -- imported from the staged
LiteGS checkout or its byte copy that ``__graft_entry__.build()`` stages under ``oracle/_ref/py`` (``oracle/build_ref.py:stage_python``)
and run on top of THIS repository's ``litegs_fused`` / ``fused_ssim`` modules and the dependency stand-ins of
``litegs_b200/shims``:

 * the reference's only in-tree correctness mechanism, ``BaseWrapper.validate()`` (fused vs pure-PyTorch script,
   wrapper.py:131-151), passes on our kernels wherever it passes on the reference's own;
 * ``litegs.render.render_preprocess`` + ``render`` + backward match the CPU oracle (image 1e-4, gradients 2e-4), with the
   reference's feedback-buffer sizing protocol (data.py:238) in both its cold and warm state;
 * with statistics running (``StatisticsHelperInst``), what the densifier reads -- fragment weight mean, fragment error
   variance, visible counts -- equals the same quantities derived from the oracle;
 * ``litegs.training.start`` trains a synthetic COLMAP scene end to end (COLMAP reader, simple_knn stand-in, cluster code,
   SparseGaussianAdam -> adamUpdate, densification -> gpu_driven_pipeline_sparse_op / statistics, PLY writer)."""
import hashlib
import json
import os
import sys

import numpy as np
import pytest
import torch

import oracle
from tests.util import PARAM_KEYS, scaled_err, small_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def litegs_ref(cuda):
    """The reference package, unmodified, on our native modules."""
    from oracle import build_ref
    path = build_ref.reference_python_path()
    if path is None:
        pytest.skip("reference Python package not available: no LiteGS checkout was found when oracle/_ref was built (oracle/build_ref.py)")
    man = os.path.join(path, "MANIFEST.json")
    if os.path.exists(man):                       # staged copy: every file is byte-identical to what was staged
        for rel, digest in json.load(open(man)).items():
            assert hashlib.sha256(open(os.path.join(path, rel), "rb").read()).hexdigest() == digest, rel
    from litegs_b200 import shims
    shims.install()
    if path not in sys.path:
        sys.path.insert(1, path)
    import litegs_fused
    import fused_ssim
    assert os.path.dirname(os.path.abspath(litegs_fused.__file__)) == ROOT and os.path.dirname(os.path.abspath(fused_ssim.__file__)) == ROOT
    import litegs
    import litegs.config
    assert os.path.abspath(litegs.__file__).startswith(os.path.abspath(path))
    assert litegs.utils.wrapper.litegs_fused is litegs_fused
    return litegs


def _ref_kernels():
    from oracle import build_ref
    return build_ref.load()


WRAPPERS = ["CreateTransformMatrix", "CreateRaySpaceTransformMatrix", "CreateCov2dDirectly", "SphericalHarmonicToRGB",
            "EighAndInverse2x2Matrix"]


def _validate_outcome(cls):
    """True / False from BaseWrapper.validate(), or the exception type when the reference's own harness breaks (two of its
    classes do on any kernels: a stale argument list in CreateRaySpaceTransformMatrix.test_inputs, wrapper.py:264-268, and
    torch.linalg.eigh refusing the 512k-matrix batch of EighAndInverse2x2Matrix.gen_inputs on this cuSOLVER)."""
    torch.manual_seed(0)
    try:
        return bool(cls.validate())
    except Exception as e:          # noqa: BLE001 -- the outcome is compared, not swallowed
        return type(e).__name__


@pytest.mark.parametrize("name", WRAPPERS)
def test_reference_validate_passes_on_our_kernels(litegs_ref, name):
    """BaseWrapper.validate(): the reference's fused-vs-script check, on our kernels; expected outcome = the outcome on the
    reference's own kernels (a check that fails or crashes on the reference's own build is not held against ours)."""
    w = litegs_ref.utils.wrapper
    cls = getattr(w, name)
    ours = _validate_outcome(cls)
    refmod = _ref_kernels()
    if refmod is None:
        assert ours is True, f"{name}.validate() -> {ours} on litegs_b200 kernels"
        return
    keep = w.litegs_fused
    w.litegs_fused = refmod
    try:
        theirs = _validate_outcome(cls)
    finally:
        w.litegs_fused = keep
    print(f"{name}.validate(): ours {ours}, reference kernels {theirs}")
    assert ours is True or ours == theirs, f"{name}.validate(): {theirs} on the reference's kernels, {ours} on ours"


def _to_torch(params, aabb, cam, dev):
    P = {k: torch.from_numpy(params[k]).to(dev).requires_grad_(True) for k in PARAM_KEYS}
    A = [torch.from_numpy(a).to(dev) for a in aabb]
    C = {k: torch.from_numpy(v).to(dev) for k, v in cam.items()}
    return P, A, C


def _oracle_case(n, hw, tile, deg, seed):
    params, aabb, cam = small_scene(n=n, hw=hw, tile=tile, sh_degree=3, seed=seed)
    rng = np.random.default_rng(seed + 100)
    w = rng.normal(size=(1, 3, hw[0], hw[1])).astype(np.float32)
    o0 = oracle.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w)
    frag = o0["fragile"][:, : hw[0], : hw[1]]
    w = w * (~frag)[:, None]
    ref = oracle.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w)
    return params, aabb, cam, w, frag, ref


@pytest.mark.parametrize("tile,deg", [((8, 16), 3), ((16, 16), 1)])
def test_reference_render_path_matches_oracle(cuda, litegs_ref, tile, deg):
    """litegs.render.render_preprocess + render (reference code, ours kernels) + backward vs the oracle; run twice so that the
    second pass sizes its buffers from the pinned feedback values written by the first (GR/compact.cu:527-549,
    GR/binning.cu:137-163 protocol, implemented host-side in litegs_b200/fused.py)."""
    L = litegs_ref
    hw = (96, 128)
    params, aabb, cam, w, frag, ref = _oracle_case(4000, hw, tile, deg, seed=11)
    nvis = int(ref["visible_chunk_id"].shape[0])
    lp, op, pp, dp = L.config.get_default_arg()
    pp.tile_size = tile
    fb_chunks = torch.zeros(4, dtype=torch.int32).pin_memory()
    fb_alloc = torch.zeros(4, dtype=torch.int32).pin_memory()
    idx = torch.tensor([2])
    wt = torch.from_numpy(w).to(cuda)
    for rnd in range(2):
        P, A, C = _to_torch(params, aabb, cam, cuda)
        ids, num, cx, cs, cr, col, cop = L.render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], P["xyz"], P["scale"], P["rot"],
                                                                    P["sh_0"], P["sh_rest"], P["opacity"], fb_chunks, idx, pp, deg)
        assert int(num.item()) == nvis and np.array_equal(ids.cpu().numpy()[:nvis], ref["visible_chunk_id"])
        img, trans, depth, normal, prim_vis = L.render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * pp.cluster_size, fb_alloc, idx,
                                                               deg, hw, pp)
        (img * wt).sum().backward()
        torch.cuda.synchronize()
        assert int(fb_chunks[2]) == nvis and int(fb_alloc[2]) == ref["sorted_pid"].shape[1]      # feedback written for the next epoch
        ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
        assert np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max() < 1e-4, rnd
        for k in PARAM_KEYS:
            g = P[k].grad
            assert type(g).__name__ == "CompactedTensor"                                           # the reference's sparse-gradient container
            cv = g.compacted_values.reshape(*ref["grads"][k].shape[:-2], -1, ref["grads"][k].shape[-1]).cpu().numpy()
            e = scaled_err(cv[..., :nvis, :], ref["grads"][k][..., :nvis, :])
            assert e < 2e-4, (rnd, k, e)


def test_reference_statistics_helper_on_our_kernels(cuda, litegs_ref):
    """enable_statistic through the reference's StatisticsHelper (statistic_helper.py:82-156, wrapper.py:501-506): the
    per-Gaussian numbers the densifier consumes (densify.py:273-292) equal the ones computed from the oracle's raster outputs."""
    L = litegs_ref
    SH = L.utils.statistic_helper.StatisticsHelperInst
    hw, tile, deg = (96, 128), (8, 16), 2
    params, aabb, cam, w, frag, ref = _oracle_case(4000, hw, tile, deg, seed=5)
    nvis = int(ref["visible_chunk_id"].shape[0])
    C_chunks, S = params["xyz"].shape[-2:]
    lp, op, pp, dp = L.config.get_default_arg()
    pp.tile_size = tile
    SH.reset(C_chunks, S, lambda epoch: True)
    P, A, C = _to_torch(params, aabb, cam, cuda)
    wt = torch.from_numpy(w).to(cuda)
    with SH.try_start(0):
        ids, num, cx, cs, cr, col, cop = L.render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], P["xyz"], P["scale"], P["rot"],
                                                                    P["sh_0"], P["sh_rest"], P["opacity"], None, None, pp, deg)
        img = L.render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * pp.cluster_size, None, None, deg, hw, pp)[0]
        (img * wt).sum().backward()
        SH.backward_callback()
    torch.cuda.synchronize()
    # expected values from the oracle: forward statistics + backward error statistic on the same lists
    o = ref
    th, tw = tile
    inter = o["inter"]
    _, _, _, fc, fw, _ = oracle.rasterize_forward(o["sorted_pid"], o["ranges"], inter["ndc"], inter["inv_cov2d"], o["color"], o["opacity"], None,
                                                  hw[0], hw[1], th, tw, enable_statistic=True)
    g_full = np.zeros_like(o["img_padded"])
    mask = (o["img_padded"][..., : hw[0], : hw[1]] >= 0) & (o["img_padded"][..., : hw[0], : hw[1]] <= 1)
    g_full[..., : hw[0], : hw[1]] = w * mask
    gmax = float(np.abs(g_full).max())
    bw = oracle.rasterize_backward(o["sorted_pid"], o["ranges"], inter["ndc"], inter["inv_cov2d"], o["color"], o["opacity"], None, o["T"],
                                   o["last"], (g_full / gmax).astype(np.float32), None, gmax, hw[0], hw[1], th, tw, enable_statistic=True,
                                   err_mode="reference")
    d_op, err_sq = bw[3], bw[5]
    ids_np = ref["visible_chunk_id"]

    def dense(a):                                       # compacted [.., nvis*S] -> dense [.., C*S] at the visible chunks
        out = np.zeros((*a.shape[:-1], C_chunks, S), a.dtype)
        out[..., ids_np, :] = a.reshape(*a.shape[:-1], -1, S)[..., :nvis, :]
        return out.reshape(*a.shape[:-1], -1)
    cnt = dense(fc[0, 0].astype(np.float64))
    exp_w_mean = dense(fw[0].astype(np.float64)) / (cnt + 1e-9)
    got_w_mean, got_cnt = SH.get_mean("fragment_weight")
    assert np.array_equal(got_cnt.cpu().numpy().astype(np.int64), cnt.astype(np.int64))
    assert scaled_err(got_w_mean.cpu().numpy(), exp_w_mean) < 2e-4
    # fragment_err: sum = d_opacity (already de-normalised), square_sum = err_sq * gmax^2  (wrapper.py:506); var as get_var()
    s1 = dense(d_op.astype(np.float64)); s2 = dense((err_sq[0] * gmax * gmax).astype(np.float64))
    exp_var = np.maximum(s2 / (cnt + 1) - (s1 / (cnt + 1)) ** 2, 0)
    got_var, _ = SH.get_var("fragment_err")
    assert scaled_err(got_var.cpu().numpy(), exp_var) < 5e-4
    # visible count per Gaussian = 1 where the splat owns at least one tile (wrapper.py:733-737 -> update_visible_count)
    _, _, alloc = oracle.get_allocate_size(inter["ndc"], inter["view_pos"][:, 2], inter["inv_cov2d"], o["opacity"], hw[0], hw[1], th, tw)
    vis = dense((alloc > 0).astype(np.int64))
    assert np.array_equal(SH.visible_count.cpu().numpy().reshape(-1).astype(np.int64), vis.reshape(-1))
    SH.reset(0, 0, lambda epoch: False)


def test_reference_trainer_runs_end_to_end(cuda, litegs_ref, tmp_path):
    """litegs.training.start (trainer.py:26-208), unmodified, on a small synthetic COLMAP scene: 24 views, 30 epochs, with
    densification active from epoch 3 -- then the saved PLY is rendered and compared with the training images."""
    L = litegs_ref
    sys.path.insert(0, os.path.join(ROOT, "examples"))
    import train_colmap
    from litegs_b200 import ply as lgs_ply, render, scene
    from litegs_b200.arguments import PipelineParams
    data = str(tmp_path / "scene")
    H, W = 135, 240
    train_colmap.make_dataset(data, n_gaussians=20_000, n_views=24, hw=(H, W), n_points=6_000, dev=cuda)
    lp, op, pp, dp = L.config.get_default_arg()
    lp.source_path = data
    lp.model_path = str(tmp_path / "out")
    lp.sh_degree = 3
    op.iterations = 24 * 30
    op.position_lr_max_steps = op.iterations
    dp.target_primitives = 12_000
    torch.manual_seed(0)
    L.training.start(lp, op, pp, dp, [], [], [], None)
    out = os.path.join(lp.model_path, "point_cloud", "finish", "point_cloud.ply")
    assert os.path.exists(out)
    g = lgs_ply.params_from_ply(out, sh_degree=3)
    n_after = g["xyz"].shape[-2] * g["xyz"].shape[-1]
    assert n_after > 6_000                                     # densification added Gaussians
    P = {k: torch.from_numpy(g[k]).to(cuda) for k in PARAM_KEYS}
    A = list(scene.cluster_aabb_torch(P["xyz"], P["scale"], P["rot"]))
    frames, _, _ = train_colmap.load_dataset(data, dev=cuda)
    ppb = PipelineParams(tile_size=(8, 16))
    mse = []
    with torch.no_grad():
        for cam, gt, _ in frames[:8]:
            img = render.render_view(A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                     P["sh_rest"], P["opacity"], 3, (H, W), ppb)[0]
            mse.append(float(((img - gt) ** 2).mean()))
    psnr = -10 * np.log10(np.mean(mse))
    print(f"reference trainer on litegs_b200 kernels: {n_after} Gaussians after 30 epochs, PSNR {psnr:.2f} dB over 8 training views")
    assert psnr > 22.0
