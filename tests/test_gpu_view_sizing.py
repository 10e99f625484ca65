"""Sizing on the GPU-driven view path (pipeline.ViewWorkspace): the device-side launch parameters, the truncation of a pair list
that outgrows its capacity, whole views at the sizing edges, and the overflow feedback to the host.

References:
  * R: numpy restatements of what lgs_view_params writes (the 8 launch parameters and the sticky word), below;
  * O: the fp64 oracle -- oracle.create_table / tileRange lists over hand-built records, and the fp64 raster over given lists;
  * S: the synchronising path (pipeline.render_view_forward / render_view_backward).  Integer state (counters, ranges, the live
    sorted_pid, last) and, in the deterministic mode, the image, T and the gradients must match it bit for bit.

Cases: zero, one and capacity +- 1 pairs; depth-key ranges of 2^k - 1 and 2^k; a run that straddles the capacity, runs longer than
the 512-pair emit window, junk past the live count; scenes seen from an identity-rotation camera, so that view-space z is world
z and the test picks the depth-key bits; a graph captured with one visible-chunk count and replayed with others; a padded image
at 12x16 tiles and 65,536 8x8 tiles (32-bit tile keys); the last populated tile closed on both paths with Level A's
CONFIG["fix_last_tile"] off; and overflow flags that land after the next batch was enqueued."""
import ctypes
import math

import numpy as np
import pytest
import torch

import oracle
from litegs_b200 import _lib, fused, pipeline, render
from litegs_b200.arguments import PipelineParams
from litegs_b200.dist import GradAccumulator
from tests import tile_cover_oracle as tc
from tests.util import PARAM_KEYS, axis_camera, deterministic, oracle_render_lists, screen_affine, tile_segments  # noqa: F401

pytestmark = pytest.mark.gpu
TILES = [(8, 16), (12, 16), (16, 16), (8, 8)]
TILE_IDS = [f"{h}x{w}" for h, w in TILES]
ptr = lambda t: ctypes.c_void_p(t.data_ptr())
stream = lambda: ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def fbits(z):
    return int(np.float32(z).view(np.uint32))


def bits_f(k):
    return float(np.uint32(k).view(np.float32))


# ---------------------------------------------------------------------------------------------------
# R: what lgs_view_params must write
# ---------------------------------------------------------------------------------------------------

def view_params_ref(counters, S, cap, planned):
    """counters (visible chunks, pairs, ~min key, max key) -> the 8 launch parameters (csrc/fused.cu, view_params_kernel)."""
    nvis, D = int(counters[0]), int(counters[1])
    kmin, kmax = ~int(counters[2]) & 0xFFFFFFFF, int(counters[3]) & 0xFFFFFFFF
    bits = max(1, (kmax - kmin).bit_length()) if (D > 0 and kmax >= kmin) else 1
    flags = (1 if D > cap else 0) | (2 if bits > planned else 0)
    as_i32 = lambda u: u - (1 << 32) if u >= (1 << 31) else u
    return [nvis * S, min(D, cap), as_i32(kmin), bits, flags, D, nvis, planned]


def sticky_ref(rows):
    """Sticky word after the views rows = [params]: |flags, max pairs, max bits, views."""
    out = [0, 0, 0, 0]
    for p in rows:
        out = [out[0] | p[4], max(out[1], p[5]), max(out[2], p[3]), out[3] + 1]
    return out


def counters_for(nvis, D, kmin, kmax):
    i32 = lambda u: u - (1 << 32) if u >= (1 << 31) else u
    return [nvis, D, i32(~kmin & 0xFFFFFFFF), i32(kmax & 0xFFFFFFFF)]


def view_params_cases():
    cap = 5000
    rows = [([0, 0, 0, 0], 32, cap, 24)]                                   # the initial (zero) counters: D = 0
    for D in (1, cap - 1, cap, cap + 1, 1 << 30):
        rows.append((counters_for(3, D, 0x3F800000, 0x3F800000 + 1000), 128, cap, 24))
    rows.append((counters_for(2, 7, 0x40000000, 0x40000000), 64, cap, 1))                  # kmin = kmax: 1 bit
    rows.append((counters_for(3, cap + 1, 0x3F000000, 0x3F000000 + (1 << 20)), 32, cap, 8))  # both flags
    for k in (7, 8, 15, 16, 23, 24, 31, 32):
        for r in ((1 << k) - 1, 1 << k):
            if r > 0xFFFFFFFF:
                continue
            kmin = 0 if k >= 31 else 0x3E800000
            for planned in (1, 8, 24, 32):
                rows.append((counters_for(5, 900, kmin, kmin + r), 96, cap, planned))
    rows.append((counters_for(4, 900, 0, 0xFFFFFFFF), 32, cap, 32))         # the full range
    return rows


def run_view_params(cuda, rows, sticky=None):
    n = len(rows)
    cnt = torch.tensor([r[0] for r in rows], dtype=torch.int32, device=cuda)
    out = torch.full((n, 8), -7, dtype=torch.int32, device=cuda)
    for i, (_, S, cap, planned) in enumerate(rows):
        _lib.call("lgs_view_params", ptr(cnt[i]), S, cap, planned, ptr(out[i]), None if sticky is None else ptr(sticky), stream())
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_view_params_match_the_restatement(cuda):
    rows = view_params_cases()
    got = run_view_params(cuda, rows)
    for i, (c, S, cap, planned) in enumerate(rows):
        assert got[i].tolist() == view_params_ref(c, S, cap, planned), (i, c, S, cap, planned, got[i].tolist())
    # every flag combination occurs
    assert {int(f) for f in got[:, 4]} == {0, 1, 2, 3}


def test_view_params_sticky_word_accumulates(cuda):
    rows = view_params_cases()
    groups = [rows[1:4], rows[3:6], rows[6:20], rows[:1], rows]
    for g in groups:
        sticky = torch.zeros(4, dtype=torch.int32, device=cuda)
        for _ in range(2):                                         # the word keeps accumulating until someone resets it
            run_view_params(cuda, g, sticky)
        want = sticky_ref([view_params_ref(*r) for r in g] * 2)
        assert sticky.cpu().tolist() == want, (sticky.cpu().tolist(), want)


# ---------------------------------------------------------------------------------------------------
# O: the truncating chain emit -> tile sort -> tile ranges on hand-built records
# ---------------------------------------------------------------------------------------------------

CHAIN_HW = (376, 504)               # > 512 tiles at every tile shape; ragged at all but 8x8
SENT = 0x5A5A                       # sentinel of the 16-bit key buffers; 32-bit buffers hold SENT * 0x10001


def chain_records(hw, tile):
    """Hand-built records (random splats, screen-sized ones with runs over several 512-pair emit windows, and splats that own no
    tile) with depths full of ties -> dict with the records, the emit order, and the oracle's full table in that order."""
    recs = np.concatenate([tc.random_cases(11, 300, hw), np.array(tc.big_cases(hw, tile, n=4))])
    H, W = hw
    off = np.array([[-1e4, -1e4, 1.0, 0.0, 1.0, 0.5], [W / 2, H / 2, 1.0, 0.0, 1.0, 0.5 / 255]])    # off-screen, too faint
    recs = np.concatenate([recs[:100], off[:1], recs[100:200], off[1:], recs[200:]])
    N = recs.shape[0]
    depth = 1.0 + ((np.arange(N) * 7919) % 37) * 1e-3                         # 37 depth values: many ties
    depth[302] = 0.5                                                          # the first run is a screen-sized splat
    inp = tc.inputs_2d(recs, hw, depth=depth)
    order = np.argsort(inp["vz"], axis=-1, kind="stable").astype(np.int64)     # depth order, ties in slot order
    th, tw = tile
    _, _, alloc = oracle.get_allocate_size(inp["ndc"], inp["vz"], inp["inv"], inp["op"], H, W, th, tw)
    prefix = np.cumsum(np.take_along_axis(alloc, order, axis=-1), axis=-1).astype(np.int32)
    total = int(prefix[0, -1])
    keys, vals = oracle.create_table(inp["ndc"], inp["inv"], inp["op"], prefix, order, total, H, W, th, tw)
    packed = np.zeros((N, 12), np.float32)
    packed[:, 2], packed[:, 3], packed[:, 4] = inp["inv"][0, 0, 0], inp["inv"][0, 0, 1], inp["inv"][0, 1, 1]
    packed[:, 5], packed[:, 9] = inp["op"][0], inp["vz"][0]
    packed[:, 10], packed[:, 11] = inp["ndc"][0, 0], inp["ndc"][0, 1]           # the emit reads the ndc centre (pad0, pad1)
    counts = np.take_along_axis(alloc, order, axis=-1)[0]
    return dict(packed=packed, order=order[0].astype(np.int32), prefix=prefix[0], counts=counts, keys=keys[0], vals=vals[0], total=total)


def expected_cut(prefix, counts, cap):
    """Length of the list the emit keeps: the start of the first run that crosses cap (all of it when none does)."""
    start = prefix - counts
    cross = np.nonzero((counts > 0) & (prefix > cap))[0]
    return int(prefix[-1]) if cross.size == 0 else int(start[cross[0]])


def run_chain(cuda, rec, hw, tile, cap, n_live, key_bits, junk=64):
    """The GPU-driven chain on the records: launch size n_live + junk with junk records, order and offsets past *n_dev, pair
    buffers larger than cap with a sentinel tail.  -> dict of the outputs (numpy)."""
    H, W = hw
    th, tw = tile
    gx, gy = -(-W // tw), -(-H // th)
    ntile = gx * gy
    N = rec["packed"].shape[0]
    rng = np.random.default_rng(cap + n_live)
    n_cap = n_live + junk
    packed = np.concatenate([rec["packed"], rng.uniform(-1, 1, (junk, 12)).astype(np.float32)])
    packed[N:, 5] = 0.9                                                       # junk that would emit if it were read
    order = np.concatenate([rec["order"][:n_live], rng.integers(0, N + junk, n_cap - n_live).astype(np.int32)])
    offs = np.concatenate([rec["prefix"][:n_live], rng.integers(0, 1 << 20, n_cap - n_live).astype(np.int32)])
    kdt = torch.int16 if key_bits == 16 else torch.int32
    sent = SENT if key_bits == 16 else SENT * 0x10001
    tail = 4096
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    keys = torch.full((cap + tail,), sent, dtype=kdt, device=cuda)
    vals = torch.full((cap + tail,), SENT * 0x10001, dtype=torch.int32, device=cuda)
    keys_s, pid = torch.full_like(keys, sent), torch.full_like(vals, SENT * 0x10001)
    ranges = torch.full((1, ntile + 2), -7, dtype=torch.int32, device=cuda)
    D = int(rec["prefix"][n_live - 1]) if n_live > 0 else 0
    vp = torch.tensor([n_live, min(D, cap)], dtype=torch.int32, device=cuda)          # *n_dev, *d_dev as lgs_view_params leaves them
    tp, to, tf = dev(packed), dev(order), dev(offs)
    nb = ctypes.c_size_t(0)
    _lib.call(f"lgs_sort_pairs_{'u16' if key_bits == 16 else 'u32'}_workspace_bytes", cap, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=cuda)
    n_dev, d_dev = ptr(vp[0]), ptr(vp[1])
    _lib.call("lgs_emit_pairs_dev", ptr(tp), ptr(tf), ptr(to), n_cap, n_dev, cap, H, W, th, tw, key_bits, ptr(keys), ptr(vals), d_dev,
              stream())
    torch.cuda.synchronize()
    emitted = (keys.cpu().numpy(), vals.cpu().numpy(), int(vp[1]))
    _lib.call("lgs_sort_pairs_u16_dev" if key_bits == 16 else "lgs_sort_pairs_u32k_dev", ptr(keys), ptr(keys_s), ptr(vals), ptr(pid), cap,
              d_dev, 0, ntile.bit_length(), ptr(ws), ctypes.c_size_t(nb.value), stream())
    _lib.call("lgs_tile_range_u16_dev" if key_bits == 16 else "lgs_tile_range_dev", ptr(keys_s), cap, d_dev, ntile, 1, ptr(ranges),
              stream())
    torch.cuda.synchronize()
    return dict(keys=emitted[0], vals=emitted[1], valid=emitted[2], keys_s=keys_s.cpu().numpy(), pid=pid.cpu().numpy(),
                ranges=ranges.cpu().numpy(), sent=sent, ntile=ntile)


def chain_caps(rec):
    """(name, cap, live splats) of the cut positions: at the end of a long run, one below it, below the first run, all pairs
    with junk past the live count, and no live splat."""
    prefix, counts = rec["prefix"], rec["counts"]
    N = prefix.shape[0]
    first = int(np.nonzero(counts)[0][0])
    assert counts[first] > 1
    big = first + 1 + int(np.argmax(counts[first + 1:]))                      # a long run after the first one
    assert counts[big] > 512
    return [("run end", int(prefix[big]), N), ("one below run end", int(prefix[big]) - 1, N), ("below first run", int(counts[first]) - 1, N),
            ("all, junk past n", int(prefix[-1]) + 3, N - 40), ("n = 0", 1000, 0)]


@pytest.mark.parametrize("key_bits", [16, 32])
@pytest.mark.parametrize("tile", TILES, ids=TILE_IDS)
def test_truncating_chain_matches_the_oracle(cuda, tile, key_bits):
    hw = CHAIN_HW
    rec = chain_records(hw, tile)
    for name, cap, n_live in chain_caps(rec):
        prefix, counts = rec["prefix"][:n_live], rec["counts"][:n_live]
        total = int(prefix[-1]) if n_live > 0 else 0
        want = expected_cut(prefix, counts, cap) if n_live > 0 else 0
        if name == "run end":
            assert want == cap < total
        elif name == "one below run end":
            assert want < cap and counts[np.searchsorted(prefix - counts, want, side="right") - 1] > 512
        elif name == "below first run":
            assert want == 0
        got = run_chain(cuda, rec, hw, tile, cap, n_live, key_bits)
        what = (name, cap, n_live, want)
        assert got["valid"] == want, (what, got["valid"])
        # expected: O's tile-sorted table restricted to the splats whose runs end at or before the cut
        order = rec["order"][:n_live]
        kept = order[(prefix <= want) & (counts > 0)]
        sel = np.isin(rec["vals"], kept)
        ek, ev = rec["keys"][sel].astype(np.int64), rec["vals"][sel]
        assert ek.size == want, what
        # the emit wrote each kept splat's run in depth order, O's tiles for it, and nothing at or past the cut
        u = lambda a: a.astype(np.int64) & (0xFFFF if key_bits == 16 else 0xFFFFFFFF)
        assert np.array_equal(got["vals"][:want], np.repeat(order, counts)[:want]), what
        srt = np.argsort(u(got["keys"][:want]), kind="stable")
        assert np.array_equal(u(got["keys"][:want])[srt], ek) and np.array_equal(got["vals"][:want][srt], ev), what
        assert (got["keys"][want:] == np.array(got["sent"]).astype(got["keys"].dtype)).all(), what
        assert (got["vals"][want:] == SENT * 0x10001).all(), what
        # the sort and the ranges: per tile, the kept splats in depth order (ties in slot order)
        assert np.array_equal(got["pid"][:want], ev), what
        assert np.array_equal(u(got["keys_s"][:want]), ek), what
        want_ranges = oracle.tileRange(ek.astype(np.int32)[None], got["ntile"], fix_last=True) if want > 0 else \
            np.concatenate([np.full((1, got["ntile"] + 1), -1, np.int32), np.zeros((1, 1), np.int32)], 1)
        assert np.array_equal(got["ranges"], want_ranges), what
        # nothing downstream wrote at or past the capacity
        for k in ("keys", "keys_s"):
            assert (got[k][cap:] == np.array(got["sent"]).astype(got[k].dtype)).all(), (what, k)
        for k in ("vals", "pid"):
            assert (got[k][cap:] == SENT * 0x10001).all(), (what, k)


# ---------------------------------------------------------------------------------------------------
# whole views on a workspace against S and O
# ---------------------------------------------------------------------------------------------------

def splat_scene(hw, px, py, z, sigma_px, opacity, chunk_of=None, seed=0):
    """Isotropic Gaussians at pixel centres (px, py) and world depths z seen from axis_camera(hw), sigma in pixels, one chunk per
    distinct chunk_of value (default: one chunk), padded with invisible Gaussians.  -> (P numpy, aabb numpy)."""
    px, py, z = (np.asarray(a, np.float64) for a in (px, py, z))
    n = px.shape[0]
    chunk_of = np.zeros(n, np.int64) if chunk_of is None else np.asarray(chunk_of)
    C = int(chunk_of.max()) + 1
    S = 32 * -(-int(np.bincount(chunk_of).max()) // 32)
    ax, bx, ay, by = screen_affine(axis_camera(hw), hw, z)
    X, Y = (px - bx) / ax, (py - by) / ay
    s = np.broadcast_to(np.asarray(sigma_px, np.float64), (n,)) / np.abs(ax)
    o = np.broadcast_to(np.asarray(opacity, np.float64), (n,))
    rng = np.random.default_rng(seed)
    xyz = np.zeros((3, C, S)); scale = np.full((3, C, S), math.log(1e-4)); rot = np.zeros((4, C, S)); rot[0] = 1.0
    opac = np.full((1, C, S), -30.0)
    fill = np.zeros(C, np.int64)
    for i in range(n):
        c = int(chunk_of[i]); j = fill[c]; fill[c] += 1
        assert j < S
        xyz[:, c, j] = X[i], Y[i], z[i]
        scale[:, c, j] = math.log(s[i])
        opac[0, c, j] = math.log(o[i] / (1 - o[i]))
    for c in range(C):                                    # padding sits on the chunk's first Gaussian
        xyz[:, c, fill[c]:] = xyz[:, c, :1]
    P = dict(xyz=xyz, scale=scale, rot=rot, sh_0=rng.uniform(-1.2, 1.2, (1, 3, C, S)), sh_rest=np.zeros((0, 3, C, S)), opacity=opac)
    P = {k: v.astype(np.float32) for k, v in P.items()}
    lo, hi = P["xyz"].min(2).astype(np.float64), P["xyz"].max(2).astype(np.float64)
    aabb = ((0.5 * (lo + hi)).astype(np.float32), (0.5 * (hi - lo) + 3 * s.max() + 1e-3).astype(np.float32))
    return P, aabb


def to_dev(cuda, P, aabb, cams):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(cuda)
    return {k: t(v) for k, v in P.items()}, [t(a) for a in aabb], [{k: t(v) for k, v in c.items()} for c in cams]


def grid_splats(hw, n, z, sigma_px, opacity=0.7, margin=0.15, seed=0):
    H, W = hw
    rng = np.random.default_rng(seed)
    return (rng.uniform(margin * W, (1 - margin) * W, n), rng.uniform(margin * H, (1 - margin) * H, n),
            np.broadcast_to(np.asarray(z, np.float64), (n,)).copy(), sigma_px, opacity)


def zeros_acc(P):
    acc = {k: torch.zeros_like(v) for k, v in P.items()}
    acc["_touched"] = torch.zeros(P["xyz"].shape[1], dtype=torch.float32, device=P["xyz"].device)
    return acc


def sync_view(P, A, cam, hw, tile, d_img):
    """S: forward and backward on the synchronising path -> (img, state, grads)."""
    img, st, _ = pipeline.render_view_forward(P, A[0], A[1], cam["frustumplane"], cam["view"], cam["proj"], 0, hw, tile, clamp_zero=True)
    acc = zeros_acc(P)
    pipeline.render_view_backward(P, st, pipeline._padded(d_img, img.shape), accumulate_into=acc, clamped_img=img)
    torch.cuda.synchronize()
    return img, st, acc


def ws_view(ws, P, A, cam, d_img):
    """One view on the workspace, its gradients into the workspace's own accumulator (fixed pointers: the backward graph's
    signature holds them)."""
    if not hasattr(ws, "test_acc"):
        ws.test_acc = zeros_acc(P)
    acc = ws.test_acc
    for v in acc.values():
        v.zero_()
    ws.forward(P, A[0], A[1], cam, 0)
    ws.backward(P, d_img, 0, acc)
    torch.cuda.synchronize()
    return acc


def assert_matches_sync(ws, img, st, acc_ws, acc_s, what):
    """Workspace state == S's, bit for bit (the gradients too: the deterministic mode is on)."""
    D = st.n_pairs
    assert torch.equal(ws.counters, st.counters), what
    vp = ws.vparams.cpu().tolist()
    assert vp == view_params_ref(st.counters.cpu().tolist(), ws.S, ws.cap, ws.planned_bits), (what, vp)
    assert vp[4] == 0, what
    # without pairs the synchronising path fills the whole range table with -1, the workspace's table ends with the list length
    # 0; no tile reads that entry then
    r = ws.ranges if D > 0 else ws.ranges[:, :-1]
    assert torch.equal(r, st.ranges[:, :r.shape[1]]) and torch.equal(ws.sorted_pid[:, :D], st.sorted_pid[:, :D]), what
    if D == 0:
        assert int(ws.ranges[0, -1]) == 0 and int(st.ranges[0, -1]) == -1
    assert torch.equal(ws.img, img) and torch.equal(ws.T, st.T) and torch.equal(ws.last, st.last), what
    for k in list(PARAM_KEYS) + ["_touched"]:
        assert torch.equal(acc_ws[k], acc_s[k]), (what, k)


def workspace_runs(ws, P, A, cams, d_img, check):
    """Every camera once eagerly, then once more (the capture run) and twice as a replay, on a side stream (graphs cannot be
    captured on the legacy default stream); check(i, acc) after each view."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for rnd in range(4):
            for i, cam in enumerate(cams):
                check(i, ws_view(ws, P, A, cam, d_img), rnd)
    torch.cuda.current_stream().wait_stream(s)


def edge_scenes(hw):
    """name -> (P, aabb, cams) of the small cases."""
    H, W = hw
    out = {}
    P, aabb = splat_scene(hw, *grid_splats(hw, 20, 4.0, 3.0))
    out["no visible chunks"] = (P, aabb, [axis_camera(hw, (0.0, 0.0, -50.0))])      # everything behind the camera
    for why, (px, py, z, o) in {"fainter than 1/255": (W / 2, H / 2, 4.0, 0.9 / 255), "z <= 0.2": (W / 2, H / 2, 0.19, 0.8),
                                "|ndc| > 1.3": (1.2 * W, H / 2, 4.0, 0.8)}.items():
        px_ = np.array([px, W * 0.3]); py_ = np.array([py, H * 0.3]); z_ = np.array([z, z]); o_ = np.array([o, o])
        if why == "|ndc| > 1.3":
            px_[1] = -0.2 * W
        P, aabb = splat_scene(hw, px_, py_, z_, 4.0, o_)
        aabb = (aabb[0], np.maximum(aabb[1], 1.0).astype(np.float32))            # the chunk is visible
        out[f"no pairs: {why}"] = (P, aabb, [axis_camera(hw)])
    P, aabb = splat_scene(hw, [W * 0.4], [H * 0.55], [3.0], 5.0, 0.8)
    out["one splat"] = (P, aabb, [axis_camera(hw)])
    P, aabb = splat_scene(hw, *grid_splats(hw, 30, 2.5, 6.0, seed=3))
    out["one depth"] = (P, aabb, [axis_camera(hw)])
    return out


@pytest.mark.parametrize("case", ["no visible chunks", "no pairs: fainter than 1/255", "no pairs: z <= 0.2", "no pairs: |ndc| > 1.3",
                                  "one splat", "one depth"])
def test_small_views_match_the_synchronising_path(cuda, deterministic, case):
    hw, tile = (64, 96), (16, 16)
    P, aabb, cams = edge_scenes(hw)[case]
    P, A, cams = to_dev(cuda, P, aabb, cams)
    d_img = torch.from_numpy(np.random.default_rng(1).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    img, st, acc_s = sync_view(P, A, cams[0], hw, tile, d_img)
    nvis, D = st.n_chunks_visible, st.n_pairs
    if case == "no visible chunks":
        assert nvis == 0 and D == 0
    elif case.startswith("no pairs"):
        assert nvis == 1 and D == 0
    else:
        assert D > 0
    if D == 0:
        assert (img == 0).all() and (st.T == 1).all() and (st.last == 0).all()
        for k in PARAM_KEYS:
            assert (acc_s[k] == 0).all(), k
    if nvis == 0:
        assert (acc_s["_touched"] == 0).all()
    if case == "one depth":
        # every splat at one depth: each tile's list is in slot order
        pid = st.sorted_pid[0, :D].cpu().numpy()
        start, end = tile_segments(st.ranges.cpu().numpy(), D)
        for t in np.nonzero(start >= 0)[0]:
            assert (np.diff(pid[start[t]:end[t]]) > 0).all(), t
        assert st.counters[2].item() == ~st.counters[3].item()      # kmin = kmax
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1024, planned_depth_bits=1)
    # the gradient buffer must stay bit-unchanged where nothing is visible: run into a buffer holding values
    workspace_runs(ws, P, A, cams, d_img, lambda i, acc, rnd: assert_matches_sync(ws, img, st, acc, acc_s, (case, rnd)))
    assert len(ws._graphs) == 2
    if nvis == 0:
        pre = {k: torch.randn_like(v) for k, v in P.items()}
        acc = {k: v.clone() for k, v in pre.items()}
        acc["_touched"] = torch.zeros(P["xyz"].shape[1], device=cuda)
        ws.forward(P, A[0], A[1], cams[0], 0)
        ws.backward(P, d_img, 0, acc)
        torch.cuda.synchronize()
        for k in PARAM_KEYS:
            assert torch.equal(acc[k], pre[k]), k
        assert (acc["_touched"] == 0).all()
    ws.post_flags()
    r = ws.check(wait=True)
    assert r == {"max_pairs": D, "max_depth_bits": 1, "views": 4 * len(cams) + (nvis == 0)}


def test_both_paths_close_the_last_tile_with_fix_last_tile_off(cuda, deterministic, monkeypatch):
    """CONFIG["fix_last_tile"] = False selects the reference's open last tile for Level A (tileRange) only: on a view whose last
    populated tile is not the grid's last, both fused paths still close it and the workspace equals S bit for bit."""
    monkeypatch.setitem(fused.CONFIG, "fix_last_tile", False)
    hw, tile = (64, 96), (16, 16)
    P, aabb, cams = edge_scenes(hw)["one splat"]
    P, A, cams = to_dev(cuda, P, aabb, cams)
    d_img = torch.from_numpy(np.random.default_rng(5).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    img, st, acc_s = sync_view(P, A, cams[0], hw, tile, d_img)
    D, r = st.n_pairs, st.ranges[0].cpu().numpy()
    ntile = r.shape[0] - 2
    top = int(np.flatnonzero((r[:ntile + 1] >= 0) & (r[:ntile + 1] < D)).max())      # highest populated (tile + 1) key
    assert 0 < D and top < ntile and r[top + 1] == D
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1024, planned_depth_bits=32)
    workspace_runs(ws, P, A, cams, d_img, lambda i, acc, rnd: assert_matches_sync(ws, img, st, acc, acc_s, rnd))


def depth_scene(hw, bits):
    """32 splats whose depth keys span exactly `bits` bits, crossing the float exponent boundary at 2.0 (8 and 16 bits) or 2.0
    and 4.0 (24 bits): keys from kmin = bits(2.0) - 2^(bits-1) to kmin + 2^bits - 1."""
    n = 32
    kmin = fbits(2.0) - (1 << (bits - 1))
    ks = kmin + np.round(np.linspace(0, (1 << bits) - 1, n)).astype(np.int64)
    ks[-1] = kmin + (1 << bits) - 1
    z = np.array([bits_f(k) for k in ks])
    rng = np.random.default_rng(bits)
    px, py = rng.uniform(0.2, 0.8, n) * hw[1], rng.uniform(0.2, 0.8, n) * hw[0]
    return splat_scene(hw, px, py, z, 4.0, 0.7, seed=bits), kmin, ks[-1]


@pytest.mark.parametrize("bits", [8, 16, 24])
def test_depth_range_at_the_planned_bits(cuda, deterministic, bits):
    """Keys spanning exactly the planned bits: no flag and S's state; planned one bit short: flagged, and check() raises with the
    measured bits.  (32 bits cannot occur in a view: the keys of positive depths above 0.2 span less than 2^31.)"""
    hw, tile = (64, 96), (8, 16)
    (P, aabb), kmin, kmax = depth_scene(hw, bits)
    P, A, cams = to_dev(cuda, P, aabb, [axis_camera(hw)])
    d_img = torch.from_numpy(np.random.default_rng(2).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    img, st, acc_s = sync_view(P, A, cams[0], hw, tile, d_img)
    c = st.counters.cpu().tolist()
    assert (~c[2] & 0xFFFFFFFF, c[3] & 0xFFFFFFFF) == (kmin, kmax)          # view z = world z exactly
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=st.n_pairs, planned_depth_bits=bits)
    workspace_runs(ws, P, A, cams, d_img, lambda i, acc, rnd: assert_matches_sync(ws, img, st, acc, acc_s, (bits, rnd)))
    ws.post_flags()
    assert ws.check(wait=True)["max_depth_bits"] == bits
    short = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=st.n_pairs, planned_depth_bits=bits - 1, use_graphs=False)
    short.forward(P, A[0], A[1], cams[0], 0)
    short.post_flags()
    torch.cuda.synchronize()
    assert short.vparams.cpu().tolist()[3:5] == [bits, 2]
    with pytest.raises(pipeline.CapacityExceeded) as e:
        short.check(wait=True)
    assert (e.value.depth_bits, e.value.planned_depth_bits) == (bits, bits - 1)


def pair_scene(hw):
    return splat_scene(hw, *grid_splats(hw, 48, np.linspace(2.0, 3.0, 48), 20.0, seed=5))


def test_pairs_at_and_one_above_capacity(cuda, deterministic):
    """cap = D: S's state.  cap = D - 1: flagged; the lists are S's restricted to the splats whose runs end before the first
    run that crosses the capacity; the emit wrote no slot past the kept length; the image is O's raster over those lists."""
    hw, tile = (192, 256), (8, 8)
    P, aabb = pair_scene(hw)
    P, A, cams = to_dev(cuda, P, aabb, [axis_camera(hw)])
    d_img = torch.from_numpy(np.random.default_rng(3).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    img, st, acc_s = sync_view(P, A, cams[0], hw, tile, d_img)
    D = st.n_pairs
    assert D >= 4096
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=D, planned_depth_bits=32)
    assert ws.cap == D
    workspace_runs(ws, P, A, cams, d_img, lambda i, acc, rnd: assert_matches_sync(ws, img, st, acc, acc_s, ("cap = D", rnd)))
    # one above: the expected cut from S's per-record counts in depth order (ties in slot order)
    packed = st.packed[0].cpu().numpy()
    tcount = st.tile_count.cpu().numpy()
    order = np.lexsort((np.arange(packed.shape[0]), np.ascontiguousarray(packed[:, 9]).view(np.uint32)))
    order = order[tcount[order] > 0]
    prefix = np.cumsum(tcount[order])
    want = expected_cut(prefix, tcount[order], D - 1)
    kept = set(order[:np.searchsorted(prefix, want, side="right")].tolist())
    assert 0 < want < D - 1
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=D - 1, planned_depth_bits=32, use_graphs=False)
    SENT32 = SENT * 0x10001
    ws.keys.fill_(SENT); ws.vals.fill_(SENT32)
    ws.forward(P, A[0], A[1], cams[0], 0)
    ws.post_flags()
    torch.cuda.synchronize()
    vp = ws.vparams.cpu().tolist()
    assert vp[1] == want and vp[4] == 1 and vp[5] == D, vp
    assert (ws.keys[want:] == SENT).all() and (ws.vals[want:] == SENT32).all()
    spid, sr = st.sorted_pid[0].cpu().numpy(), st.ranges.cpu().numpy()
    s0, e0 = tile_segments(sr, D)
    s1, e1 = tile_segments(ws.ranges.cpu().numpy(), want)
    pid = ws.sorted_pid[0, :want].cpu().numpy()
    lists, n_pairs = [], 0
    for t in range(len(s0)):
        full = spid[s0[t]:e0[t]] if s0[t] >= 0 else spid[:0]
        exp = np.array([i for i in full.tolist() if i in kept], np.int32)
        got = pid[s1[t]:e1[t]] if s1[t] >= 0 else pid[:0]
        assert np.array_equal(got, exp), t
        lists.append(exp); n_pairs += exp.size
    assert n_pairs == want
    with pytest.raises(pipeline.CapacityExceeded) as e:
        ws.check(wait=True)
    assert (e.value.pairs, e.value.pair_capacity) == (D, D - 1)
    # the image: O's raster over the truncated lists
    H, W = hw
    oimg, oT, frag = oracle_render_lists(ws.packed[0].cpu().numpy(), pid[None], ws.ranges.cpu().numpy(), hw, tile)
    mask = frag[:H, :W]
    assert mask.mean() < 0.02
    err = np.abs(ws.img[0, :, :H, :W].cpu().numpy() - oimg[:, :H, :W])[:, ~mask].max()
    terr = np.abs(ws.T[0, 0, :H, :W].cpu().numpy() - oT[:H, :W])[~mask].max()
    print(f"truncated view: {want} of {D} pairs kept, |img - O| {err:.2e}, |T - O| {terr:.2e}, masked {mask.mean():.4f}")
    assert err < 1e-4 and terr < 1e-4


def chunk_row_scene(hw, n_chunks=8, per_chunk=12):
    """n_chunks clusters of Gaussians in a row along x at z in [4, 4.6); seen from axis_camera(hw, (tx, 0, 0))."""
    W = hw[1]
    px, py, z, ch = [], [], [], []
    rng = np.random.default_rng(9)
    for c in range(n_chunks):
        cx = W * (0.1 + 0.8 * c / (n_chunks - 1))
        px += list(cx + rng.uniform(-3, 3, per_chunk)); py += list(hw[0] * rng.uniform(0.3, 0.7, per_chunk))
        z += list(rng.uniform(4.0, 4.6, per_chunk)); ch += [c] * per_chunk
    return splat_scene(hw, np.array(px), np.array(py), np.array(z), 3.0, 0.8, chunk_of=np.array(ch))


@pytest.mark.parametrize("hw,tile", [((64, 96), (16, 16)), ((100, 120), (12, 16)), ((2048, 2048), (8, 8))],
                         ids=["64x96-16x16", "padded-12x16", "2048-8x8-32bit-keys"])
def test_graph_replayed_over_visible_chunk_counts(cuda, deterministic, hw, tile):
    """Captured with few visible chunks, replayed with all, none and few again: each replay equals S for its own camera."""
    P, aabb = chunk_row_scene(hw)
    W = hw[1]
    ax = screen_affine(axis_camera(hw), hw, np.array([4.3]))[0][0]
    few, all_, none = axis_camera(hw, (-0.55 * W / ax, 0.0, 0.0)), axis_camera(hw), axis_camera(hw, (0.0, 0.0, -50.0))
    P, A, cams = to_dev(cuda, P, aabb, [few, few, all_, none, few])
    d_img = torch.from_numpy(np.random.default_rng(4).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    refs = [sync_view(P, A, c, hw, tile, d_img) for c in cams]
    nvis = [r[1].n_chunks_visible for r in refs]
    assert 0 < nvis[0] < 8 and nvis[2] == 8 and nvis[3] == 0, nvis
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=max(r[1].n_pairs for r in refs), planned_depth_bits=24)
    assert ws.u16 == (hw != (2048, 2048))
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for i, cam in enumerate(cams):                   # eager, capture, then replays
            acc = ws_view(ws, P, A, cam, d_img)
            assert_matches_sync(ws, *refs[i], acc, (hw, i))
            assert len(ws._graphs) == (0 if i == 0 else 2)
    torch.cuda.current_stream().wait_stream(s)


# ---------------------------------------------------------------------------------------------------
# the feedback protocol
# ---------------------------------------------------------------------------------------------------

def batch_scene(cuda, hw):
    """One scene, three cameras with different pair counts and depth ranges (the camera's z offset shrinks the depth-key ulps)."""
    P, aabb = splat_scene(hw, *grid_splats(hw, 40, np.linspace(5.0, 5.0 + 2.5e-5, 40), 4.0, margin=0.45, seed=7))
    cams = [axis_camera(hw), axis_camera(hw, (0.0, 0.0, -4.3)), axis_camera(hw, (0.0, 0.0, -2.5))]
    return to_dev(cuda, P, aabb, cams)


def measured_bits(P, A, cams, hw, tile):
    """Depth-key bits of each camera's view on the synchronising path."""
    out = []
    for c in cams:
        _, st, _ = pipeline.render_view_forward(P, A[0], A[1], c["frustumplane"], c["view"], c["proj"], 0, hw, tile)
        out.append(view_params_ref(st.counters.cpu().tolist(), 32, 1 << 20, 32)[3])
    return out


def test_check_folds_a_batch(cuda):
    hw, tile = (64, 96), (16, 16)
    P, A, cams = batch_scene(cuda, hw)
    rows = []
    for c in cams:
        _, st, _ = pipeline.render_view_forward(P, A[0], A[1], c["frustumplane"], c["view"], c["proj"], 0, hw, tile)
        rows.append(view_params_ref(st.counters.cpu().tolist(), 32, 1 << 20, 32))
    want = sticky_ref(rows)
    assert len({r[3] for r in rows}) == 3 and len({r[5] for r in rows}) >= 2, rows
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1 << 20, planned_depth_bits=32, use_graphs=False)
    for c in cams:
        ws.forward(P, A[0], A[1], c, 0)
    ws.post_flags()
    assert ws.check(wait=True) == {"max_pairs": want[1], "max_depth_bits": want[2], "views": 3}
    assert ws.check(wait=True) is None
    # two posts read by one check: folded
    for c in cams[:2]:
        ws.forward(P, A[0], A[1], c, 0)
        ws.post_flags()
    two = sticky_ref(rows[:2])
    assert ws.check(wait=True) == {"max_pairs": two[1], "max_depth_bits": two[2], "views": 2}


@pytest.mark.parametrize("where", [0, 1, 2])
def test_overflow_in_any_view_of_a_batch_raises(cuda, where):
    hw, tile = (64, 96), (16, 16)
    P, A, cams = batch_scene(cuda, hw)
    bits = []
    for c in cams:
        _, st, _ = pipeline.render_view_forward(P, A[0], A[1], c["frustumplane"], c["view"], c["proj"], 0, hw, tile)
        bits.append(view_params_ref(st.counters.cpu().tolist(), 32, 1 << 20, 32)[3])
    deep = int(np.argmax(bits))
    planned = sorted(bits)[-2]                              # only the deepest camera overflows
    order = [i for i in range(3) if i != deep]
    order.insert(where, deep)
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1 << 20, planned_depth_bits=planned)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        for rnd in range(3):                                # eager, capture, replay
            for i in order:
                ws.forward(P, A[0], A[1], cams[i], 0)
            ws.post_flags()
            with pytest.raises(pipeline.CapacityExceeded) as e:
                ws.check(wait=True)
            assert e.value.depth_bits == bits[deep] > planned
    torch.cuda.current_stream().wait_stream(s)


SLEEP_CYCLES = 150_000_000          # ~76 ms at 1980 MHz: holds the stream while the host enqueues the next batch


def test_late_flags_are_not_lost(cuda):
    """An overflowing batch whose flags cannot land before the next batch is enqueued (the stream is held by a short timed
    kernel), then a clean batch: the overflow is still reported."""
    hw, tile = (64, 96), (16, 16)
    P, A, cams = batch_scene(cuda, hw)
    assert measured_bits(P, A, cams, hw, tile) == [6, 9, 7]
    ws = pipeline.ViewWorkspace(P, hw, tile, pair_capacity=1 << 20, planned_depth_bits=8, use_graphs=False)
    for c in cams:                                          # warm up: camera 1 needs 9 depth-key bits, the others fewer
        ws.forward(P, A[0], A[1], c, 0)
    ws.post_flags()
    with pytest.raises(pipeline.CapacityExceeded) as e:
        ws.check(wait=True)
    assert e.value.depth_bits == 9
    torch.cuda.synchronize()
    with pytest.raises(pipeline.CapacityExceeded) as e:
        torch.cuda._sleep(SLEEP_CYCLES)
        ws.forward(P, A[0], A[1], cams[1], 0)               # this batch overflows the planned depth bits ...
        ws.post_flags()
        ws.check(wait=False)                                # what render_views does at the start of the next batch
        ws.forward(P, A[0], A[1], cams[0], 0)               # ... and this one does not
        ws.post_flags()
        torch.cuda.synchronize()
        ws.check(wait=True)
    assert (e.value.depth_bits, e.value.planned_depth_bits) == (9, 8)


def render_batch(P, A, cams, hw, pp, acc, views, n_streams, w):
    acc.zero_()
    losses = render.render_views(len(views), lambda i: cams[views[i]], lambda i, img: (img * w).sum(), A[0], A[1], P["xyz"], P["scale"],
                                 P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 0, hw, pp, acc.grads(), n_streams=n_streams)
    torch.cuda.synchronize()
    return [float(x) for x in losses], {k: v.clone() for k, v in acc.grads().items()}


@pytest.mark.parametrize("n_streams", [1, 3])
def test_render_views_reports_late_flags_and_remeasures(cuda, deterministic, n_streams):
    """Through render_views: the probe batch sizes the workspaces on camera 0 (6 depth-key bits, 8 planned); after the eager and
    the capture batch, a replayed batch with camera 1 (9 bits) overflows them while the stream is held; a clean batch follows;
    check_views must raise.  The next batch
    measures again on the synchronising path, and the one after that, on fresh workspaces, equals S."""
    hw = (64, 96)
    P, A, cams = batch_scene(cuda, hw)
    pp = PipelineParams(tile_size=(16, 16))
    acc = GradAccumulator(P)
    w = torch.from_numpy(np.random.default_rng(0).normal(size=(1, 3, *hw)).astype(np.float32)).to(cuda)
    clean, deep = [0, 0, 0], [0, 1, 0]
    assert measured_bits(P, A, cams, hw, (16, 16)) == [6, 9, 7]
    render.reset_view_workspaces()
    keep = pipeline.SYNC_FREE
    try:
        pipeline.SYNC_FREE = False
        ref = render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)
        pipeline.SYNC_FREE = True
        render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)          # probe: measures the sizes
        ent = next(iter(render._slot_cache.values()))
        assert ent.bits == 8 and ent.ws == []
        render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)          # eager on the workspaces
        render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)          # captures the graphs (a capture synchronises the device)
        with pytest.raises(pipeline.CapacityExceeded):
            torch.cuda._sleep(SLEEP_CYCLES)
            render.render_views(len(deep), lambda i: cams[deep[i]], lambda i, img: (img * w).sum(), A[0], A[1], P["xyz"], P["scale"],
                                P["rot"], P["sh_0"], P["sh_rest"], P["opacity"], 0, hw, pp, acc.grads(), n_streams=n_streams)
            render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)
            render.check_views(wait=True)
        assert ent.ws is None
        render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)          # measures again (synchronising)
        assert ent.ws == [] and ent.bits == 8
        got = render_batch(P, A, cams, hw, pp, acc, clean, n_streams, w)    # fresh workspaces
        assert len(ent.ws) == n_streams
        render.check_views(wait=True)
    finally:
        pipeline.SYNC_FREE = keep
        render.reset_view_workspaces()
    assert got[0] == ref[0]
    for k in list(PARAM_KEYS) + ["_touched"]:
        assert torch.equal(got[1][k], ref[1][k]), k
