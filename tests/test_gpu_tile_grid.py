"""Tile grids at 4K and on both sides of every tile-key width boundary, against the CPU oracle.

The fused pipeline stores the (tile + 1) sort keys in 16 bits while tiles + 1 < 65536 and in 32 bits beyond.  4K at 8x16 tiles
(the C4 grid, 64,800 tiles) puts keys above 32767 into the 16-bit path, whose top bit a sign extension or a truncation would
lose; 4K at 8x8 (129,600 tiles) needs 17 key bits.  The cases:

    C4 grid          8x16  3840x2160  64,800 tiles   16-bit keys, more than 8 << 20 pairs (the tile sort takes cub's onesweep)
    last 16-bit      8x16  3470x2410  65,534 tiles   16-bit keys up to 0xFFFE (both edges ragged)
    first 32-bit     8x16  4075x2050  65,535 tiles   32-bit keys, key 0xFFFF populated
    4K at 8x8        8x8   3840x2160 129,600 tiles   32-bit keys, 17 key bits

For each: the synchronising pipeline against the oracle (tile lists, contributor counts, image, six gradients), the GPU-driven
ViewWorkspace against the synchronising pipeline, and the tile-range kernels of both key widths against oracle.tileRange on
key lists built to cross 32767/32768 and 65535/65536."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, pipeline, render, scene
from litegs_b200.arguments import PipelineParams
from tests.util import PARAM_KEYS, differing_tiles, scaled_err, tile_segments

pytestmark = pytest.mark.gpu

C4_LOG_SCALES = (0.002 * np.exp(-0.5), 0.02 * np.exp(-0.5))       # BASELINE.md: C4 shifts the log-scales by -0.5
SPARSE_LOG_SCALES = (0.003, 0.02)

# name, tile (h, w), image (h, w), Gaussians, cube half-size, log-scale range, seed, 16-bit keys, check of the highest key
CASES = [
    ("c4_grid", (8, 16), (2160, 3840), 620_000, 1.0, C4_LOG_SCALES, 0, True, lambda top, ntile: top >= 0x8000),
    ("last_u16", (8, 16), (2410, 3470), 50_000, 1.5, SPARSE_LOG_SCALES, 1, True, lambda top, ntile: top == ntile == 0xFFFE),
    ("first_u32", (8, 16), (2050, 4075), 50_000, 1.5, SPARSE_LOG_SCALES, 2, False, lambda top, ntile: top == ntile == 0xFFFF),
    ("4k_8x8", (8, 8), (2160, 3840), 50_000, 1.5, SPARSE_LOG_SCALES, 3, False, lambda top, ntile: top > 0xFFFF),
]
IDS = [c[0] for c in CASES]


@functools.lru_cache(maxsize=None)
def _inputs(name):
    _, tile, hw, n, cube, lsr, seed, _, _ = next(c for c in CASES if c[0] == name)
    p = scene.make_scene(n, sh_degree=3, seed=seed, cube=cube, log_scale_range=lsr)
    params = {k: p[k] for k in PARAM_KEYS}
    return params, (p["cluster_origin"], p["cluster_extend"]), scene.make_camera(0, 64, hw[1], hw[0])


def _to_cuda(params, aabb, cam, dev, grad=False):
    P = {k: torch.from_numpy(params[k]).to(dev).requires_grad_(grad) for k in PARAM_KEYS}
    return P, [torch.from_numpy(a).to(dev) for a in aabb], {k: torch.from_numpy(v).to(dev) for k, v in cam.items()}


def _top_key(ranges, n):
    """Highest populated (tile + 1) key of a range table."""
    start, end = tile_segments(ranges, n)
    return int(np.flatnonzero((start >= 0) & (end > start)).max()) + 1


@pytest.mark.parametrize("name,tile,hw,n,cube,lsr,seed,u16,top_ok", CASES, ids=IDS)
def test_view_matches_oracle(cuda, name, tile, hw, n, cube, lsr, seed, u16, top_ok):
    """The method of test_gpu_fullsize.py::test_c2_one_view_matches_oracle at this grid: tile lists equal to the oracle's up to
    corner-grazing pairs (at most 1e-5 of the pairs), contributor counts bit-exact and the image within 1e-4 off the fragile
    pixels, the six gradients within 2e-4 with zero loss weight on fragile pixels and on the tiles whose lists differ."""
    H, W = hw
    deg = 3
    params, aabb, cam = _inputs(name)
    w = np.random.default_rng(7).normal(size=(1, 3, H, W)).astype(np.float32)
    o0 = oracle.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w)
    frag = o0["fragile"][:, :H, :W].copy()
    P, A, C = _to_cuda(params, aabb, cam, cuda, grad=True)
    with torch.no_grad():
        _, st, _ = pipeline.render_view_forward({k: P[k].detach() for k in PARAM_KEYS}, A[0], A[1], C["frustumplane"], C["view"],
                                                C["proj"], deg, hw, tile)
    ntile = st.ranges.shape[1] - 2
    D = o0["sorted_pid"].shape[1]
    ranges = st.ranges.cpu().numpy()
    top = _top_key(ranges, st.n_pairs)
    bad, npairs = differing_tiles(ranges, st.sorted_pid.cpu().numpy(), o0["ranges"], o0["sorted_pid"])
    assert ((ntile + 1) < 65536) == u16
    assert top_ok(top, ntile), (top, ntile)
    if name == "c4_grid":
        assert st.n_pairs > (8 << 20)              # the automatic choice of the tile sort takes cub's onesweep here
    assert abs(st.n_pairs - D) <= 1e-5 * D and npairs <= 1e-5 * D, (st.n_pairs, D, npairs)
    gx = -(-W // tile[1])
    for t in bad:
        ty, tx = divmod(int(t), gx)
        frag[:, ty * tile[0]:(ty + 1) * tile[0], tx * tile[1]:(tx + 1) * tile[1]] = True
    # The blend stops once T <= 1/8192.  Rows below the middle of a 4K frame sit at ndc + 1 in [1, 2), where fp32 rounds the pixel
    # position twice as coarsely as above, and after ~100 blended splats the two transmittances differ by a few 1e-4 of T (99.99th
    # percentile 2.9e-4 there, 1.9e-4 above the middle, on the C4 grid): wider than the oracle's own margin on that threshold
    # (1e-8 = 8e-5 of 1/8192).  A pixel whose final T, on either side, lies within 5e-4 of 1/8192 stopped on the threshold and
    # counts as fragile too (about 0.1 % of the pixels).  The same frame at 16x16 tiles, whose keys stay below 32768, differs on
    # the same pixels without this: the cause is the rounding, not the key width.
    on_stop = lambda T: np.abs(T[:, 0, :H, :W] * 8192.0 - 1.0) < 5e-4
    frag |= on_stop(st.T.cpu().numpy()) | on_stop(o0["T"])
    print(f"{name}: {ntile} tiles, D = {D} pairs (ours {st.n_pairs}), highest key {top}, {len(bad)} tiles / {npairs} pairs differ "
          f"from the oracle's lists, {frag.sum()} fragile pixels ({frag.mean() * 100:.2f} %)")
    assert frag.mean() < 0.10
    lc = st.last.cpu().numpy()[:, 0, :H, :W].astype(np.uint16)
    assert np.array_equal(lc[~frag], o0["last"][:, 0, :H, :W].astype(np.uint16)[~frag])
    w = w * (~frag)[:, None]
    ref = oracle.render_forward_backward(params, aabb, cam, hw, tile, deg, lambda img: w)
    pp = PipelineParams(tile_size=tile)
    img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], P["xyz"], P["scale"], P["rot"], P["sh_0"], P["sh_rest"],
                             P["opacity"], deg, hw, pp)[0]
    (img * torch.from_numpy(w).to(cuda)).sum().backward()
    ok = ~np.broadcast_to(frag[:, None], ref["img"].shape)
    err = np.abs(img.detach().cpu().numpy()[ok] - ref["img"][ok]).max()
    assert err < 1e-4, err
    nvis = int(ref["visible_chunk_id"].shape[0])
    for k in PARAM_KEYS:
        g = P[k].grad.compacted_values.cpu().numpy()[..., :nvis, :].astype(np.float64)
        r = ref["grads"][k][..., :nvis, :].astype(np.float64)
        e = float(np.abs(g - r).max() / np.abs(r).max())
        print(f"   d {k}: max|diff| / max|ref| = {e:.2e}")
        assert e < 2e-4, (k, e)


@pytest.mark.parametrize("name,tile,hw,n,cube,lsr,seed,u16,top_ok", CASES, ids=IDS)
def test_workspace_matches_synchronising_path(cuda, name, tile, hw, n, cube, lsr, seed, u16, top_ok):
    """The GPU-driven path (device-side counts: lgs_emit_pairs_dev, lgs_sort_pairs_u16_dev / lgs_sort_pairs_u32k_dev,
    lgs_tile_range_u16_dev / lgs_tile_range_dev) against pipeline.render_view_forward / render_view_backward: tile lists,
    image, transmittance and contributor counts bit for bit, accumulated gradients within 1e-5."""
    H, W = hw
    params, aabb, cam = _inputs(name)
    P, A, C = _to_cuda(params, aabb, cam, cuda)
    img_ref, st, _ = pipeline.render_view_forward(P, A[0], A[1], C["frustumplane"], C["view"], C["proj"], 3, hw, tile, clamp_zero=True)
    D = st.n_pairs
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=int(D * 1.3), planned_depth_bits=32, use_graphs=False)
    assert ws.u16 == u16
    img = ws.forward(P, A[0], A[1], C, 3)
    torch.cuda.synchronize()
    assert int(ws.vparams[5]) == D
    assert torch.equal(ws.ranges, st.ranges)
    assert torch.equal(ws.sorted_pid[:, :D], st.sorted_pid)
    assert torch.equal(img, img_ref) and torch.equal(ws.T, st.T) and torch.equal(ws.last, st.last)
    d_img = torch.zeros_like(img_ref)
    d_img[..., :H, :W] = torch.randn((1, 3, H, W), generator=torch.Generator(device="cpu").manual_seed(4)).to(cuda)
    got = {k: torch.zeros_like(P[k]) for k in PARAM_KEYS}
    want = {k: torch.zeros_like(P[k]) for k in PARAM_KEYS}
    ws.backward(P, d_img, 3, got)
    pipeline.render_view_backward(P, st, d_img, accumulate_into=want, clamped_img=img_ref)
    torch.cuda.synchronize()
    for k in PARAM_KEYS:
        e = scaled_err(got[k].cpu().numpy(), want[k].cpu().numpy())
        assert e < 1e-5, (k, e)


def test_level_a_equals_level_b_at_4k_8x8(cuda):
    """Level A (render_preprocess + render: lgs_create_table with int32 keys, lgs_tile_range) against Level B (the fused
    pipeline) at 129,600 tiles, as test_gpu_fullsize.py::test_c2_level_a_equals_level_b does at 1080p."""
    name, tile, hw = "4k_8x8", (8, 8), (2160, 3840)
    H, W = hw
    params, aabb, cam = _inputs(name)
    P, A, C = _to_cuda(params, aabb, cam, cuda)
    pp = PipelineParams(tile_size=tile)
    w = torch.randn((1, 3, H, W), generator=torch.Generator(device="cpu").manual_seed(2)).to(cuda)
    outs = []
    for level in ("A", "B"):
        Q = {k: v.clone().requires_grad_(True) for k, v in P.items()}
        if level == "A":
            ids, num, cx, cs, cr, col, cop = render.render_preprocess(A[0], A[1], C["frustumplane"], C["view"], Q["xyz"], Q["scale"],
                                                                      Q["rot"], Q["sh_0"], Q["sh_rest"], Q["opacity"], None, None, pp, 3)
            img = render.render(C["view"], C["proj"], cx, cs, cr, col, cop, num * 128, None, None, 3, hw, pp)[0]
        else:
            img = render.render_view(A[0], A[1], C["frustumplane"], C["view"], C["proj"], Q["xyz"], Q["scale"], Q["rot"], Q["sh_0"],
                                     Q["sh_rest"], Q["opacity"], 3, hw, pp)[0]
        (img * w).sum().backward()
        outs.append((img.detach(), {k: Q[k].grad.compacted_values for k in PARAM_KEYS}))
    assert float(outs[0][0].abs().max()) > 0
    assert float((outs[0][0] - outs[1][0]).abs().max()) < 2e-5
    for k in PARAM_KEYS:
        a, b = outs[0][1][k], outs[1][1][k]
        assert float((a - b).abs().max()) / (float(a.abs().max()) + 1e-30) < 2e-4, k


# ---- tile ranges on their own -------------------------------------------------------------------------------------------

def _key_list(rng, max_tile, first, last):
    """Sorted (tile + 1) keys in [1, max_tile]: about half the tiles populated at random, dense runs across 32767/32768 and
    65535/65536 (where the grid reaches them) with empty tiles between them, and tile 1 / tile max_tile populated or not."""
    keys = rng.integers(1, max_tile + 1, size=max_tile // 2)
    cross = []
    for b in (0x8000, 0x10000):
        cross += [b - 9] * 2 + list(range(b - 4, b + 3)) * 3 + [b + 5] * 4
    keys = np.concatenate([keys, np.array(cross)])
    keys = keys[(keys >= 1) & (keys <= max_tile)]
    keys = keys[(keys != 1) & (keys != max_tile)]
    keys = np.concatenate([keys, [1] * 3 * first, [max_tile] * 2 * last])
    return np.sort(keys).astype(np.int32)


def _tile_range(cuda, keys, max_tile, fix_last, u16, dev_form):
    """One call of lgs_tile_range / _dev / _u16_dev on `keys`; the _dev forms get a larger capacity whose tail holds garbage
    (unsorted keys) that a kernel reading past *length_dev would pick up."""
    L = keys.shape[0]
    buf = keys
    if dev_form:
        junk = np.random.default_rng(L).integers(0, max_tile + 1, size=L // 3 + 777).astype(np.int32)
        buf = np.concatenate([keys, junk])
    k = torch.from_numpy(buf.astype(np.uint16).view(np.int16) if u16 else buf).to(cuda)
    out = torch.full((1, max_tile + 2), -7, dtype=torch.int32, device=cuda)
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    sfx = "_u16" if u16 else ""
    if dev_form:
        n_dev = torch.tensor([L], dtype=torch.int32, device=cuda)
        _lib.call(f"lgs_tile_range{sfx}_dev", k.data_ptr(), buf.shape[0], n_dev.data_ptr(), max_tile, fix_last, out.data_ptr(), st)
    else:
        _lib.call(f"lgs_tile_range{sfx}", k.data_ptr(), 1, L, max_tile, fix_last, out.data_ptr(), st)
    torch.cuda.synchronize()
    return out.cpu().numpy()


# the 16-bit keys have the device-length form only
RANGE_CASES = [(u16, max_tile, dev_form) for dev_form in (False, True) for u16, max_tile in
               [(True, 64_800), (True, 65_534), (False, 64_800), (False, 65_534), (False, 65_535), (False, 129_600)] if dev_form or not u16]


@pytest.mark.parametrize("u16,max_tile,dev_form", RANGE_CASES,
                         ids=[f"{u}-{m}-{'device_length' if d else 'host_length'}" for u, m, d in RANGE_CASES])
def test_tile_range_matches_oracle(cuda, u16, max_tile, dev_form):
    rng = np.random.default_rng(max_tile + 7 * u16)
    for first in (0, 1):
        for last in (0, 1):
            keys = _key_list(rng, max_tile, first, last)
            for fix_last in (0, 1):
                got = _tile_range(cuda, keys, max_tile, fix_last, u16, dev_form)
                want = oracle.tileRange(keys[None], max_tile, fix_last=bool(fix_last))
                bad = np.flatnonzero(got[0] != want[0])
                assert bad.size == 0, (first, last, fix_last, bad[:8], got[0, bad[:8]], want[0, bad[:8]])
    for key in sorted({1, 0x7FFF, 0x8000, min(0xFFFF, max_tile), max_tile}):      # a single-key list
        for fix_last in (0, 1):
            keys = np.array([key], np.int32)
            got = _tile_range(cuda, keys, max_tile, fix_last, u16, dev_form)
            assert np.array_equal(got, oracle.tileRange(keys[None], max_tile, fix_last=bool(fix_last))), (key, fix_last)


def test_16bit_key_guards_of_the_device_forms(cuda):
    """65,535 tiles do not fit the 16-bit keys (tiles + 1 < 65536): the 16-bit forms refuse them, 65,534 tiles pass."""
    st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    i32 = lambda *v: torch.tensor(v, dtype=torch.int32, device=cuda)
    keys, vals, ranges = i32(0, 0), i32(0, 0), torch.empty(65_537, dtype=torch.int32, device=cuda)
    packed = torch.zeros((1, 1, 12), dtype=torch.float32, device=cuda)
    offsets, order, n_dev = i32(0), i32(0), i32(1)           # one splat that owns no pair: emission has nothing to write
    for max_tile, ok in ((65_534, True), (65_535, False)):
        args = (keys.data_ptr(), 1, n_dev.data_ptr(), max_tile, 1, ranges.data_ptr(), st)
        if ok:
            _lib.call("lgs_tile_range_u16_dev", *args)
        else:
            with pytest.raises(_lib.LiteGSB200Error):
                _lib.call("lgs_tile_range_u16_dev", *args)
    for (H, W), ok in (((2410, 3470), True), ((2050, 4075), False)):          # 65,534 and 65,535 tiles of 8x16
        args = (packed.data_ptr(), offsets.data_ptr(), order.data_ptr(), 1, n_dev.data_ptr(), 1, H, W, 8, 16, 16, keys.data_ptr(),
                vals.data_ptr(), None, st)
        if ok:
            _lib.call("lgs_emit_pairs_dev", *args)
        else:
            with pytest.raises(_lib.LiteGSB200Error):
                _lib.call("lgs_emit_pairs_dev", *args)
    torch.cuda.synchronize()
