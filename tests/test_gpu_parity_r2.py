"""GPU parity tests closing the holes the round-1 review listed (VERDICT "What's weak" 1, 3): every compiled variant of the
raster kernels (enable_statistic, enable_trans, specific_tiles, both backward kernels), the SH->RGB op and the
cluster_size=0 path of render_preprocess, the eigenvectors of the 2x2 eigendecomposition, the tile order, and the
reference's err_square_sum recurrence -- all against the CPU oracle on identical seeded inputs, through the C ABI."""
import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, fused, render, wrapper
from litegs_b200.arguments import PipelineParams
from tests.util import PARAM_KEYS, oracle_projected, raster_case, rel_err, scaled_err, small_scene

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


# ---------------------------------------------------------------------------------------------------
# SphericalHarmonicToRGB (GR/transform.cu:951-1361, wrapper.py:526-566) and the cluster_size=0 path
# ---------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("deg", [0, 1, 2, 3])
def test_sh2rgb_forward_backward(cuda, deg):
    rng = np.random.default_rng(deg)
    N, V, R = 1537, 1, 15                       # N not a multiple of the block size; sh_rest always has 15 rows (sh_degree 3 storage)
    sh0 = rng.normal(size=(1, 3, N)).astype(np.float32)
    shr = (0.3 * rng.normal(size=(R, 3, N))).astype(np.float32)
    d = rng.normal(size=(V, 3, N)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    got = fused.sh2rgb_forward(deg, T(sh0, cuda), T(shr, cuda), T(d, cuda)).cpu().numpy()
    ref = oracle.sh2rgb_forward(deg, sh0, shr, d)
    assert rel_err(got, ref) < TOL
    # the pure-PyTorch form the reference checks its kernel against (utils/spherical_harmonics.py:38-93, restated in fp64)
    g = rng.normal(size=(V, 3, N)).astype(np.float32)
    g0, gr, gd = fused.sh2rgb_backward(deg, T(g, cuda), R, T(d, cuda), T(sh0, cuda), T(shr, cuda))
    o0, orr, _ = oracle.sh2rgb_backward(deg, g, R, d)
    K = (deg + 1) ** 2
    assert scaled_err(g0.cpu().numpy(), o0) < TOL
    assert scaled_err(gr.cpu().numpy()[: K - 1], orr[: K - 1]) < TOL if K > 1 else True
    assert float(gr[K - 1:].abs().max()) == 0.0 if K - 1 < R else True       # rows above the active degree read as zero
    assert float(gd.abs().max()) == 0.0                                        # direction gradient dropped (GR/transform.cu:1288-1290)


def test_sh2rgb_autograd_wrapper_matches_fd(cuda):
    """wrapper.SphericalHarmonicToRGB.call_fused is differentiable in sh_0 / sh_rest: compare with the analytic basis."""
    rng = np.random.default_rng(7)
    N = 300
    sh0 = torch.from_numpy(rng.normal(size=(1, 3, N)).astype(np.float32)).to(cuda).requires_grad_(True)
    shr = torch.from_numpy(rng.normal(size=(15, 3, N)).astype(np.float32)).to(cuda).requires_grad_(True)
    d = rng.normal(size=(1, 3, N)).astype(np.float32)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    w = rng.normal(size=(1, 3, N)).astype(np.float32)
    rgb = wrapper.SphericalHarmonicToRGB.call_fused(3, sh0, shr, T(d, cuda))
    (rgb * T(w, cuda)).sum().backward()
    raw = oracle.sh2rgb_forward(3, sh0.detach().cpu().numpy(), shr.detach().cpu().numpy(), d)
    assert (raw < 0).any() and float(rgb.min()) == 0.0            # the wrapper clamps at 0 (wrapper.py:558) ...
    o0, orr, _ = oracle.sh2rgb_backward(3, w * (raw > 0), 15, d)  # ... and the clamp blocks the gradient there
    assert scaled_err(sh0.grad.cpu().numpy(), o0) < TOL and scaled_err(shr.grad.cpu().numpy(), orr) < TOL


def _oracle_unclustered(flat, cam, hw, tile, deg, w):
    """Oracle for the cluster_size = 0 path (litegs/render/__init__.py:36-46): PyTorch-style activation (true derivatives),
    SH -> RGB through the sh2rgb op with the clamp at 0 of wrapper.py:558, then the common projection / binning / raster chain."""
    H, W = hw
    th, tw = tile
    xyz, sc_raw, q_raw, sh0, shr, o_raw = (flat[k] for k in PARAM_KEYS)
    N = xyz.shape[-1]
    xyz4 = np.concatenate([xyz, np.ones((1, N), np.float32)], 0)
    scale = np.exp(sc_raw)
    qn = np.maximum(np.sqrt((q_raw * q_raw).sum(0, keepdims=True)), 1e-12)
    rot = q_raw / qn
    opacity = 1.0 / (1.0 + np.exp(-o_raw))
    V = cam["view"][0]
    center = -(V[3:4, :3] @ V[:3, :3].T)                                   # [1,3]
    dirs = xyz[None] - center.T[None]
    dirs = dirs / np.maximum(np.sqrt((dirs * dirs).sum(1, keepdims=True)), 1e-12)
    raw = oracle.sh2rgb_forward(deg, sh0, shr, dirs.astype(np.float32))
    color = np.maximum(raw, 0)
    inter = oracle.project(xyz4, scale, rot, cam["view"], cam["proj"], hw)
    ranges, pid, _, _ = oracle.binning(inter["ndc"], inter["view_pos"][:, 2], inter["inv_cov2d"], opacity, None, hw, tile, True)
    img, T_, last, _, _, fragile = oracle.rasterize_forward(pid, ranges, inter["ndc"], inter["inv_cov2d"], color, opacity, None, H, W, th, tw)
    out = dict(img=np.clip(img[..., :H, :W], 0, 1), fragile=fragile)
    if w is None:
        return out
    g_full = np.zeros_like(img)
    mask = (img[..., :H, :W] >= 0) & (img[..., :H, :W] <= 1)
    g_full[..., :H, :W] = w * mask
    gmax = float(np.abs(g_full).max())
    d_ndc, d_cov, d_col, d_op, _, _ = oracle.rasterize_backward(pid, ranges, inter["ndc"], inter["inv_cov2d"], color, opacity, None, T_, last,
                                                                (g_full / gmax).astype(np.float32), None, gmax, H, W, th, tw)
    gp, gs, gq = oracle.project_backward(inter, d_ndc, d_cov, scale, rot, cam["view"], cam["proj"])
    g0, gr, _ = oracle.sh2rgb_backward(deg, (d_col * (raw > 0)).astype(np.float32), shr.shape[0], dirs.astype(np.float32))
    dot = (gq * rot).sum(0, keepdims=True)
    out["grads"] = dict(xyz=gp[:3], scale=gs * scale, rot=(gq - dot * rot) / qn, sh_0=g0, sh_rest=gr,
                        opacity=d_op * opacity * (1 - opacity))
    return out


@pytest.mark.parametrize("deg", [0, 3])
def test_render_without_clusters_matches_oracle(cuda, deg):
    """render_preprocess / render with cluster_size = 0 (litegs/render/__init__.py:36-46): activation in PyTorch, SH through
    sh2rgb_forward/backward (clamped at 0), everything else identical."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=3000, hw=hw, tile=tile, seed=21)
    flat_np = {k: params[k].reshape(*params[k].shape[:-2], -1).copy() for k in PARAM_KEYS}
    rng = np.random.default_rng(5)
    w = rng.normal(size=(1, 3, *hw)).astype(np.float32)
    frag = _oracle_unclustered(flat_np, cam, hw, tile, deg, None)["fragile"][:, : hw[0], : hw[1]]
    w = w * (~frag)[:, None]
    ref = _oracle_unclustered(flat_np, cam, hw, tile, deg, w)
    flat = {k: torch.from_numpy(flat_np[k]).to(cuda).requires_grad_(True) for k in PARAM_KEYS}
    C = {k: torch.from_numpy(v).to(cuda) for k, v in cam.items()}
    pp = PipelineParams(tile_size=tile, cluster_size=0, sparse_grad=False)
    ids, num, cx, cs, cr, col, cop = render.render_preprocess(None, None, C["frustumplane"], C["view"], flat["xyz"], flat["scale"], flat["rot"],
                                                              flat["sh_0"], flat["sh_rest"], flat["opacity"], None, None, pp, deg)
    assert ids is None and num is None
    img = render.render(C["view"], C["proj"], cx, cs, cr, col, cop, None, None, None, deg, hw, pp)[0]
    (img * T(w, cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    assert np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max() < TOL
    for k in PARAM_KEYS:
        e = scaled_err(flat[k].grad.cpu().numpy(), ref["grads"][k])
        assert e < 2e-4, (k, e)


# ---------------------------------------------------------------------------------------------------
# EighAndInverse2x2Matrix: eigenvectors (GR/transform.cu:1364-1454)
# ---------------------------------------------------------------------------------------------------

def test_eigenvectors(cuda, proj):
    cov = proj["o"]["cov2d"]
    val, vec, inv = fused.eigh_and_inv_2x2matrix_forward(T(cov, cuda), None)
    oval, ovec, oinv = oracle.eigh_and_inv_2x2matrix_forward(cov)
    val, vec = val.cpu().numpy().astype(np.float64), vec.cpu().numpy().astype(np.float64)
    # vec[b, i, k, n] = component i of eigenvector k (columns are the vectors, as torch.linalg.eigh: GR/transform.cu:1411-1412).
    # The same vectors as the oracle, up to the sign ambiguity of an eigenvector
    s = np.sign((vec * ovec).sum(axis=1, keepdims=True))
    s[s == 0] = 1
    close = np.abs(vec * s - ovec).max(axis=(1, 2))
    gap = np.abs(oval[:, 0] - oval[:, 1]) / np.maximum(np.abs(oval).max(axis=1), 1e-30)
    assert (close[gap > 1e-3] < 5e-4).all()                  # well separated eigenvalues: vectors agree
    # and they ARE eigenvectors: cov v_k = lambda_k v_k, unit length, orthogonal
    c = cov.astype(np.float64)
    for k in range(2):
        v = vec[:, :, k]                                     # [V,2,N]
        cv = np.stack([c[:, 0, 0] * v[:, 0] + c[:, 0, 1] * v[:, 1], c[:, 1, 0] * v[:, 0] + c[:, 1, 1] * v[:, 1]], axis=1)
        res = np.abs(cv - val[:, k][:, None] * v).max(axis=1) / np.maximum(np.abs(val).max(axis=1), 1e-30)
        assert res.max() < 2e-4, res.max()
        assert np.abs((v * v).sum(axis=1) - 1).max() < 1e-4
    assert np.abs((vec[:, :, 0] * vec[:, :, 1]).sum(axis=1)).max() < 1e-4


# ---------------------------------------------------------------------------------------------------
# raster variants: statistics, transmittance gradient, specific tiles, both backward kernels
# ---------------------------------------------------------------------------------------------------

def _lists(proj, tile):
    o, hw = proj["o"], proj["hw"]
    ranges, sorted_pid, _, _ = oracle.binning(o["ndc"], o["view_pos"][:, 2], o["inv_cov2d"], o["opacity"], None, hw, tile)
    return ranges, sorted_pid


@pytest.mark.parametrize("bwd", [1, 2])
@pytest.mark.parametrize("tile", [(8, 16), (16, 16), (12, 16), (8, 8)])
def test_raster_backward_kernels_default_flags(cuda, proj, tile, bwd):
    """Both backward kernels (scalar v1, packed-pair v2) against the oracle on the oracle's own forward state."""
    _lib.call("lgs_set_backward_kernel", bwd)
    try:
        raster_case(cuda, proj, tile, "cpasync")
    finally:
        _lib.call("lgs_set_backward_kernel", 2)


@pytest.mark.parametrize("tile", [(8, 16), (16, 16)])
def test_raster_statistics_forward(cuda, proj, tile):
    """enable_statistic: fragment_count (exact) and fragment_weight_sum per splat (GR/raster.cu:273-301)."""
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, pid = _lists(proj, tile)
    oimg, oT, olast, ofc, ofw, fragile = oracle.rasterize_forward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None,
                                                                  hw[0], hw[1], th, tw, enable_statistic=True, fragile_eps=2e-6)
    out = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                  T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, True, False, False)
    img, Tr, _, last, packed, fc, fw = out
    fc, fw = fc.cpu().numpy(), fw.cpu().numpy()
    # a fragile pixel may count one fragment more or less: bound the disagreement by the number of fragile pixels
    diff = np.abs(fc.astype(np.int64) - ofc.astype(np.int64))
    assert diff.sum() <= 2 * int(fragile.sum()) + 0, (diff.sum(), fragile.sum())
    same = diff[0, 0] == 0
    assert same.mean() > 0.99
    assert scaled_err(fw[0, 0][same], ofw[0, 0][same]) < 2e-4
    # the image is the same with and without statistics
    img0 = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                   T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, False, False, False)[0]
    assert torch.equal(img, img0)


def _backward_inputs(proj, tile, seed=1, with_trans=False):
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, pid = _lists(proj, tile)
    oimg, oT, olast, _, _, fragile = oracle.rasterize_forward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None,
                                                               hw[0], hw[1], th, tw, fragile_eps=2e-6)
    rng = np.random.default_rng(seed)
    g = rng.normal(size=oimg.shape).astype(np.float32)
    g[np.broadcast_to(fragile[:, None], g.shape)] = 0.0
    gt = None
    if with_trans:
        gt = rng.normal(size=oT.shape).astype(np.float32)
        gt[fragile[:, None]] = 0.0
    return ranges, pid, oT, olast, g, gt, fragile


@pytest.mark.parametrize("bwd", [1, 2])
@pytest.mark.parametrize("tile", [(8, 16), (16, 16), (12, 16), (8, 8)])
def test_raster_backward_with_transmittance_gradient(cuda, proj, tile, bwd):
    """enable_trans: dL/dT_final enters d alpha (GR/raster.cu:771-774)."""
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, pid, oT, olast, g, gt, _ = _backward_inputs(proj, tile, with_trans=True)
    gmax = float(np.abs(g).max())
    ref = oracle.rasterize_backward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast, g / gmax, gt / gmax,
                                    gmax, hw[0], hw[1], th, tw)
    packed = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                     T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, False, True, False)[4]
    _lib.call("lgs_set_backward_kernel", bwd)
    try:
        got = fused.rasterize_backward(T(pid, cuda), T(ranges, cuda), packed, None, T(oT, cuda), T(olast, cuda), T(g / gmax, cuda),
                                       T(gt / gmax, cuda), None, torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, False)
    finally:
        _lib.call("lgs_set_backward_kernel", 2)
    for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
        assert scaled_err(a.cpu().numpy(), b) < TOL, (name, scaled_err(a.cpu().numpy(), b))
    # and it differs from the gradient without the transmittance term (the flag is live)
    ref0 = oracle.rasterize_backward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast, g / gmax, None,
                                     gmax, hw[0], hw[1], th, tw)
    assert scaled_err(ref[3], ref0[3]) > 1e-2


@pytest.mark.parametrize("mode", ["reference", "pixel"])
@pytest.mark.parametrize("tile", [(8, 16), (16, 16), (12, 16), (8, 8)])
def test_raster_backward_statistics(cuda, proj, tile, mode):
    """enable_statistic in the backward: err_square_sum per splat -- the reference's lane-running recurrence
    (GR/raster.cu:779-784, default) and the per-pixel form -- plus unchanged gradients."""
    o, hw = proj["o"], proj["hw"]
    th, tw = tile
    ranges, pid, oT, olast, g, _, _ = _backward_inputs(proj, tile, seed=3)
    gmax = float(np.abs(g).max())
    ref = oracle.rasterize_backward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast, g / gmax, None,
                                    gmax, hw[0], hw[1], th, tw, enable_statistic=True, err_mode=mode)
    packed = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                     T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, True, False, False)[4]
    _lib.call("lgs_set_err_square_mode", 1 if mode == "reference" else 0)
    try:
        got = fused.rasterize_backward(T(pid, cuda), T(ranges, cuda), packed, None, T(oT, cuda), T(olast, cuda), T(g / gmax, cuda), None, None,
                                       torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, True)
    finally:
        _lib.call("lgs_set_err_square_mode", 1)
    for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
        assert scaled_err(a.cpu().numpy(), b) < TOL, (name, scaled_err(a.cpu().numpy(), b))
    e, oe = got[5].cpu().numpy(), ref[5]
    assert oe.max() > 0
    assert scaled_err(e, oe) < 2e-4, scaled_err(e, oe)
    assert float(got[4].abs().max()) == 0.0                   # err_sum is allocated and left at zero (GR/raster.cu:816 commented out)


@pytest.mark.parametrize("bwd", [1, 2])
def test_raster_specific_tiles(cuda, proj, bwd):
    """specific_tiles: only the listed tiles are rendered / differentiated, in the given order, 0 entries are skipped
    (GR/raster.cu:184-196,623-634); everything else reads as empty."""
    o, hw = proj["o"], proj["hw"]
    tile = (8, 16)
    th, tw = tile
    ranges, pid = _lists(proj, tile)
    gx, gy = (hw[1] + tw - 1) // tw, (hw[0] + th - 1) // th
    rng = np.random.default_rng(2)
    sel = rng.permutation(gx * gy)[: (gx * gy) // 3].astype(np.int32) + 1
    sel = np.concatenate([sel, np.zeros(3, np.int32)])[None]              # with padding entries
    oimg, oT, olast, _, _, fragile = oracle.rasterize_forward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], sel,
                                                               hw[0], hw[1], th, tw, fragile_eps=2e-6)
    out = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                  T(o["opacity"], cuda), T(sel, cuda), hw[0], hw[1], th, tw, False, False, False)
    img, Tr, _, last, packed, _, _ = out
    ok = ~fragile
    m3 = np.broadcast_to(ok[:, None], oimg.shape)
    assert rel_err(img.cpu().numpy()[m3], oimg[m3]) < TOL
    assert np.array_equal(last.cpu().numpy()[:, 0][ok], olast[:, 0][ok])
    # tiles not listed are black with T = 1
    tmask = np.zeros(gx * gy + 1, bool); tmask[sel[0]] = True; tmask[0] = False
    tm = np.repeat(np.repeat(tmask[1:].reshape(gy, gx), th, 0), tw, 1)
    assert float(np.abs(img.cpu().numpy()[0][:, ~tm]).max()) == 0.0 and float(np.abs(Tr.cpu().numpy()[0, 0][~tm] - 1).max()) == 0.0
    g = rng.normal(size=oimg.shape).astype(np.float32)
    g[np.broadcast_to(fragile[:, None], g.shape)] = 0.0
    gmax = float(np.abs(g).max())
    ref = oracle.rasterize_backward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], sel, oT, olast, g / gmax, None, gmax,
                                    hw[0], hw[1], th, tw)
    _lib.call("lgs_set_backward_kernel", bwd)
    try:
        got = fused.rasterize_backward(T(pid, cuda), T(ranges, cuda), packed, T(sel, cuda), T(oT, cuda), T(olast, cuda), T(g / gmax, cuda), None,
                                       None, torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, False)
    finally:
        _lib.call("lgs_set_backward_kernel", 2)
    for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
        assert scaled_err(a.cpu().numpy(), b) < TOL, (name, scaled_err(a.cpu().numpy(), b))


def test_tile_order_is_a_descending_permutation(cuda):
    rng = np.random.default_rng(0)
    for ntile in (16200, 64800, 129600):                     # 1080p at 8x16 tiles, 4K at 8x16 and at 8x8
        work = np.minimum(rng.exponential(300, size=(2, ntile)), 9000).astype(np.int32)
        work[:, ::7] = 0
        order = torch.empty((2, ntile), dtype=torch.int32, device=cuda)
        w = T(work, cuda)
        _lib.call("lgs_tile_order", w.data_ptr(), 2, ntile, order.data_ptr(), torch.cuda.current_stream().cuda_stream)
        od = order.cpu().numpy()
        for b in range(2):
            assert np.array_equal(np.sort(od[b]), np.arange(1, ntile + 1)), ntile    # a permutation of the 1-based tile ids
            wb = np.minimum(work[b][od[b] - 1] >> 2, 1023)
            assert (np.diff(wb) <= 0).all(), ntile                                # non-increasing in the bucketed work


def test_fused_pipeline_tile_order_changes_nothing(cuda):
    """Level B with and without the heaviest-first tile order: same image (bit for bit), same gradients up to the order of
    the fp32 atomics."""
    hw, tile = (96, 128), (8, 16)
    params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=11)
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    pp = PipelineParams(tile_size=tile)
    res = []
    for flag in (True, False):
        fused.CONFIG["tile_order"] = flag
        try:
            P = {k: torch.from_numpy(params[k]).to(cuda).requires_grad_(True) for k in PARAM_KEYS}
            A = [torch.from_numpy(a).to(cuda) for a in aabb]
            C = {k: torch.from_numpy(v).to(cuda) for k, v in cam.items()}
            img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"],
                                     P["sh_rest"], P["opacity"], 3, hw, pp)[0]
            (img * w).sum().backward()
            res.append((img.detach().clone(), {k: P[k].grad.compacted_values.clone() for k in PARAM_KEYS}))
        finally:
            fused.CONFIG["tile_order"] = True
    assert torch.equal(res[0][0], res[1][0])
    for k in PARAM_KEYS:
        assert scaled_err(res[0][1][k].cpu().numpy(), res[1][1][k].cpu().numpy()) < 1e-5, k


def test_last_contributor_is_unsigned_16_bit(cuda):
    """A pixel that stays active through more than 32767 list entries: the count is stored as an unsigned 16-bit value and the
    backward walks the whole list (the reference reads the tensor as unsigned short, GR/raster.cu:683-686)."""
    hw, tile = (8, 16), (8, 16)
    n = 40000
    rng = np.random.default_rng(0)
    # n faint splats (alpha below 1/256 is still VISITED while the pixel is active: the count increases, nothing is blended),
    # the last one opaque
    ndc = np.zeros((1, 4, n), np.float32); ndc[:, 3] = 1
    ndc[0, 0] = rng.uniform(-0.5, 0.5, n); ndc[0, 1] = rng.uniform(-0.5, 0.5, n)
    inv = np.zeros((1, 2, 2, n), np.float32); inv[0, 0, 0] = 0.02; inv[0, 1, 1] = 0.02
    col = rng.uniform(0.2, 0.8, (1, 3, n)).astype(np.float32)
    op = np.full((1, n), 0.003, np.float32)            # alpha < 1/256 everywhere: visited (the count increases) but never blended
    op[0, -1] = 0.9
    pid = np.arange(n, dtype=np.int32)[None]
    ranges = np.array([[-1, 0, n]], np.int32)
    oimg, oT, olast, _, _, fragile = oracle.rasterize_forward(pid, ranges, ndc, inv, col, op, None, hw[0], hw[1], 8, 16, fragile_eps=1e-7)
    assert int(olast.astype(np.uint16).max()) == n
    out = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(ndc, cuda), T(inv, cuda), T(col, cuda), T(op, cuda), None, hw[0], hw[1],
                                  8, 16, False, False, False)
    img, Tr, _, last, packed, _, _ = out
    assert np.array_equal(last.cpu().numpy().astype(np.uint16), olast.astype(np.uint16))
    ok = ~fragile
    m3 = np.broadcast_to(ok[:, None], oimg.shape)
    assert rel_err(img.cpu().numpy()[m3], oimg[m3]) < TOL
    g = rng.normal(size=oimg.shape).astype(np.float32)
    g[np.broadcast_to(fragile[:, None], g.shape)] = 0.0
    ref = oracle.rasterize_backward(pid, ranges, ndc, inv, col, op, None, oT, olast, g, None, 1.0, hw[0], hw[1], 8, 16)
    for bwd in (1, 2):
        _lib.call("lgs_set_backward_kernel", bwd)
        try:
            got = fused.rasterize_backward(T(pid, cuda), T(ranges, cuda), packed, None, T(oT, cuda), T(olast, cuda), T(g, cuda), None, None,
                                           torch.tensor([1.0], device=cuda), hw[0], hw[1], 8, 16, False)
        finally:
            _lib.call("lgs_set_backward_kernel", 2)
        # the opaque splat sits at list position 39999: a signed 16-bit read would never reach it
        assert abs(float(got[3][0, -1])) > 0
        for a, b, name in zip(got[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
            assert scaled_err(a.cpu().numpy(), b) < 2e-4, (bwd, name, scaled_err(a.cpu().numpy(), b))


def test_deterministic_backward_is_bit_identical(cuda, proj):
    """lgs_set_deterministic(1): the backward accumulates the per-(tile, splat) sums as 64-bit fixed point with integer atomics,
    so the gradients of two runs are bit-identical (and still match the oracle); the default fp32 RED path is only reproducible to
    rounding.  Checked on the op level (oracle forward state) and through the fused pipeline with its unordered tile buckets."""
    o, hw = proj["o"], proj["hw"]
    tile = (8, 16)
    th, tw = tile
    ranges, pid, oT, olast, g, _, _ = _backward_inputs(proj, tile, seed=9)
    gmax = float(np.abs(g).max())
    ref = oracle.rasterize_backward(pid, ranges, o["ndc"], o["inv_cov2d"], o["color"], o["opacity"], None, oT, olast, g / gmax, None, gmax,
                                    hw[0], hw[1], th, tw)
    packed = fused.rasterize_forward(T(pid, cuda), T(ranges, cuda), T(o["ndc"], cuda), T(o["inv_cov2d"], cuda), T(o["color"], cuda),
                                     T(o["opacity"], cuda), None, hw[0], hw[1], th, tw, False, False, False)[4]

    def run():
        return fused.rasterize_backward(T(pid, cuda), T(ranges, cuda), packed, None, T(oT, cuda), T(olast, cuda), T(g / gmax, cuda), None, None,
                                        torch.tensor([gmax], device=cuda), hw[0], hw[1], th, tw, False)
    _lib.call("lgs_set_deterministic", 1)
    try:
        a, b = run(), run()
        for x, y, r, name in zip(a[:4], b[:4], ref[:4], ("d_ndc", "d_cov2d_inv", "d_color", "d_opacity")):
            assert torch.equal(x, y), name
            assert scaled_err(x.cpu().numpy(), r) < TOL, name
        # fused pipeline, 4000 Gaussians: forward + backward twice from scratch
        params, aabb, cam = small_scene(n=4000, hw=hw, tile=tile, seed=11)
        w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
        pp = PipelineParams(tile_size=tile)
        res = []
        for _ in range(2):
            P = {k: torch.from_numpy(params[k]).to(cuda).requires_grad_(True) for k in PARAM_KEYS}
            A = [torch.from_numpy(x).to(cuda) for x in aabb]
            C = {k: torch.from_numpy(v).to(cuda) for k, v in cam.items()}
            img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                                     P["opacity"], 3, hw, pp)[0]
            (img * w).sum().backward()
            res.append({k: P[k].grad.compacted_values.clone() for k in PARAM_KEYS})
        for k in PARAM_KEYS:
            assert torch.equal(res[0][k], res[1][k]), k
    finally:
        _lib.call("lgs_set_deterministic", 0)
