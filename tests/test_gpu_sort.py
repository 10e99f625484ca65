"""GPU tests of the stable LSD radix sort behind lgs_sort_pairs_u16/_u32 (both implementations, and the automatic choice
between them) against torch's stable sort on the same bit range: keys AND payload order must be identical (integer work:
bit-exact).  Covers the shapes the pipeline uses (14/16 tile bits on u16 keys, 17 tile bits and 24/32 depth bits on u32 keys,
more than 8 << 20 tile keys where the automatic choice switches to cub), ragged tails, single-element and empty inputs, a
sub-range of bits, a constant key (every key in one digit), and the device-side-count entry points of the GPU-driven path."""
import ctypes

import pytest
import torch

from litegs_b200 import _lib

pytestmark = pytest.mark.gpu


# implementation -> (lgs_set_sort_impl, lgs_set_radix_form): the own sort's histogram / row-scan / scatter passes (the default
# form), its onesweep form, cub, and the automatic per-call choice (-1: nothing forced)
IMPLS = {"lgs": (1, 0), "lgs_onesweep": (1, 1), "cub": (0, 0), "auto": (-1, 0)}


def _force(impl):
    _lib.call("lgs_set_sort_impl", IMPLS[impl][0])
    _lib.call("lgs_set_radix_form", IMPLS[impl][1])


def _unforce():
    _lib.call("lgs_set_sort_impl", -1)
    _lib.call("lgs_set_radix_form", 0)


def _sort(keys, vals, begin, end, impl):
    dev = keys.device
    n = keys.numel()
    u16 = keys.dtype == torch.int16
    sfx = "_u16" if u16 else "_u32"
    nb = ctypes.c_size_t(0)
    _lib.call(f"lgs_sort_pairs{sfx}_workspace_bytes", max(n, 1), ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    ko, vo = torch.full_like(keys, -1), torch.full_like(vals, -1)
    _force(impl)
    try:
        _lib.call(f"lgs_sort_pairs{sfx}", ctypes.c_void_p(keys.data_ptr()), ctypes.c_void_p(ko.data_ptr()), ctypes.c_void_p(vals.data_ptr()),
                  ctypes.c_void_p(vo.data_ptr()), n, begin, end, ctypes.c_void_p(ws.data_ptr()), ctypes.c_size_t(nb.value),
                  ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    finally:
        _unforce()
    torch.cuda.synchronize()
    return ko, vo


def _expect(keys, vals, begin, end):
    k = keys.to(torch.int64) & (0xFFFF if keys.dtype == torch.int16 else 0xFFFFFFFF)
    digit = (k >> begin) & ((1 << (end - begin)) - 1)
    order = torch.sort(digit, stable=True).indices
    return keys[order], vals[order]


CASES = [  # dtype, n, begin, end, key generator
    (torch.int16, 1, 0, 14, "uniform"), (torch.int16, 100, 0, 14, "uniform"), (torch.int16, 2048, 0, 14, "uniform"),
    (torch.int16, 2049, 0, 16, "uniform"), (torch.int16, 1_000_003, 0, 14, "uniform"), (torch.int16, 5_000_001, 0, 14, "runs"),
    (torch.int16, 4_194_305, 0, 13, "uniform"), (torch.int16, 300_000, 3, 11, "uniform"), (torch.int16, 70_000, 0, 9, "uniform"),
    (torch.int32, 1, 0, 32, "uniform"), (torch.int32, 4097, 0, 32, "uniform"), (torch.int32, 1_000_064, 0, 32, "depth"),
    (torch.int32, 1_000_064, 0, 24, "depth"), (torch.int32, 5_000_000, 0, 32, "depth"), (torch.int32, 123_457, 5, 22, "uniform"),
    (torch.int32, 50_000, 0, 32, "constant"), (torch.int32, 50_000, 0, 0, "uniform"),
    # tile keys of 4K frames: 16 bits at 8x16 tiles, 17 bits at 8x8, more than 8 << 20 pairs
    (torch.int16, 8_500_003, 0, 16, "runs"), (torch.int32, 8_600_001, 0, 17, "runs"),
]


@pytest.mark.parametrize("impl", list(IMPLS))
@pytest.mark.parametrize("dtype,n,begin,end,kind", CASES)
def test_sort_pairs_matches_stable_sort(cuda, impl, dtype, n, begin, end, kind):
    g = torch.Generator(device="cpu").manual_seed(n + 31 * end)
    hi = 1 << (16 if dtype == torch.int16 else 32)
    if kind == "uniform":
        k = torch.randint(0, hi, (n,), generator=g, dtype=torch.int64)
    elif kind == "runs":                       # what emit produces: short runs of consecutive tile ids, over the whole key range
        start = torch.randint(1, (1 << end) - 6, (n // 7 + 1,), generator=g, dtype=torch.int64)
        k = (start[:, None] + torch.arange(7)[None, :]).reshape(-1)[:n]
    elif kind == "depth":                      # float bits of view-space z in [0.2, 6): top byte almost constant
        z = torch.rand(n, generator=g) * 5.8 + 0.2
        k = z.view(torch.int32).to(torch.int64)
        k[::17] = 0xFFFFFFFF                   # culled splats carry the all-ones key
    else:
        k = torch.full((n,), 0x40490FDB, dtype=torch.int64)
    if dtype == torch.int16:
        keys = (k & 0xFFFF).to(torch.int32).to(torch.int16)     # wraps to the signed view of the same bits
    else:
        keys = torch.where(k >= (1 << 31), k - (1 << 32), k).to(torch.int32)
    vals = torch.arange(n, dtype=torch.int32)
    keys, vals = keys.to(cuda), vals.to(cuda)
    ko, vo = _sort(keys, vals, begin, end, impl)
    ek, ev = _expect(keys, vals, begin, end)
    assert torch.equal(vo, ev), f"payload order differs at {int((vo != ev).nonzero()[0])}"
    assert torch.equal(ko, ek)


@pytest.mark.parametrize("junk", [0, 40_000], ids=["capacity_is_count", "junk_past_count"])
@pytest.mark.parametrize("impl", list(IMPLS))
def test_device_count_depth_sort_orders_keys_inside_the_range(cuda, impl, junk):
    """lgs_sort_pairs_u32_dev, the depth sort of both view paths: keys inside [*bias_dev, *bias_dev + 2^bits) come out in full-key
    stable order; the keys outside (culled splats, all ones) may land anywhere but must all still be present.  The launch covers
    the live count plus `junk` unsorted slots past *n_dev (the synchronising path launches exactly the count, the workspace a
    capacity); forcing cub (LGS_SORT) does not reach this sort: it is the own radix sort in every setting."""
    g = torch.Generator(device="cpu").manual_seed(7)
    n = 700_001
    z = torch.rand(n, generator=g) * 3.4 + 1.3                       # crosses the 2.0 and 4.0 exponent boundaries
    k = z.view(torch.int32).to(torch.int64)
    k[::11] = 0xFFFFFFFF
    inside = k != 0xFFFFFFFF
    kmin, kmax = int(k[inside].min()), int(k[inside].max())
    bits = max(1, (kmax - kmin).bit_length())
    assert bits <= 24 < (kmin ^ kmax).bit_length()
    tail = torch.randint(0, 1 << 31, (junk,), generator=g, dtype=torch.int64)
    keys = torch.cat([torch.where(k >= (1 << 31), k - (1 << 32), k), tail]).to(torch.int32).to(cuda)
    vals = torch.cat([torch.arange(n), tail]).to(torch.int32).to(cuda)
    cap = n + junk
    nb = ctypes.c_size_t(0)
    _lib.call("lgs_sort_pairs_u32_workspace_bytes", cap, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=cuda)
    ko, vo = torch.empty_like(keys), torch.empty_like(vals)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    bias_dev = torch.tensor([kmin], dtype=torch.int32, device=cuda)          # positive float bits: below 2^31
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    _force(impl)
    try:
        _lib.call("lgs_sort_pairs_u32_dev", ptr(keys), ptr(ko), ptr(vals), ptr(vo), cap, ptr(n_dev), ptr(bias_dev), bits, ptr(ws),
                  ctypes.c_size_t(nb.value), None)
    finally:
        _unforce()
    torch.cuda.synchronize()
    vo_c, ko_c = vo[:n].cpu().long(), ko[:n].cpu()
    assert torch.equal(torch.sort(vo_c).values, torch.arange(n))      # a permutation of the live slots
    assert torch.equal(ko_c.long() & 0xFFFFFFFF, k[vo_c])              # keys travel with their payload
    got = vo_c[inside[vo_c]]                                           # order of the keys that matter
    want = torch.sort(torch.where(inside, k, torch.full_like(k, 1 << 40)), stable=True).indices[: int(inside.sum())]
    assert torch.equal(got, want)


@pytest.mark.parametrize("capacity,n", [(300_000, 123_457), (9_000_000, 8_500_001)])
@pytest.mark.parametrize("form", ["passes", "onesweep"])
@pytest.mark.parametrize("entry", ["lgs_sort_pairs_u16_dev", "lgs_sort_pairs_u32k_dev", "lgs_sort_pairs_u32_dev"])
def test_device_count_sorts_sort_the_live_prefix(cuda, entry, form, capacity, n):
    """The GPU-driven entry points launch for `capacity` items and read the live count from *n_dev (and, for the rebased depth
    sort, the key bias from *bias_dev): the first *n_dev outputs are the stable sort of the first *n_dev inputs, and the
    unsorted garbage after them in the input changes nothing.  u16: tile keys of 16 bits; u32k: tile keys of 17 bits (4K at
    8x8); u32: depth keys, 24 bits above a bias."""
    g = torch.Generator(device="cpu").manual_seed(capacity + len(entry))
    if entry == "lgs_sort_pairs_u32_dev":
        bias, bits = 0x3FA00000, 24                                      # float bits of 1.25, keys up to 1.25 + 2^24 ulps
        live = bias + torch.randint(0, 1 << bits, (n,), generator=g, dtype=torch.int64)
    else:
        bits = 16 if entry == "lgs_sort_pairs_u16_dev" else 17
        start = torch.randint(1, (1 << bits) - 6, (n // 7 + 1,), generator=g, dtype=torch.int64)
        live = (start[:, None] + torch.arange(7)[None, :]).reshape(-1)[:n]
    junk = torch.randint(0, 1 << 31, (capacity - n,), generator=g, dtype=torch.int64)
    k = torch.cat([live, junk])
    u16 = entry == "lgs_sort_pairs_u16_dev"
    keys = ((k & 0xFFFF).to(torch.int32).to(torch.int16) if u16 else k.to(torch.int32)).to(cuda)
    vals = torch.cat([torch.arange(n, dtype=torch.int32), torch.randint(0, 1 << 30, (capacity - n,), generator=g, dtype=torch.int32)]).to(cuda)
    nb = ctypes.c_size_t(0)
    _lib.call(f"lgs_sort_pairs_{'u16' if u16 else 'u32'}_workspace_bytes", capacity, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=cuda)
    ko, vo = torch.full_like(keys, -1), torch.full_like(vals, -1)
    n_dev = torch.tensor([n], dtype=torch.int32, device=cuda)
    ptr = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.call("lgs_set_radix_form", 1 if form == "onesweep" else 0)
    try:
        if entry == "lgs_sort_pairs_u32_dev":
            bias_dev = torch.tensor([bias], dtype=torch.int32, device=cuda)
            _lib.call(entry, ptr(keys), ptr(ko), ptr(vals), ptr(vo), capacity, ptr(n_dev), ptr(bias_dev), bits, ptr(ws),
                      ctypes.c_size_t(nb.value), None)
        else:
            _lib.call(entry, ptr(keys), ptr(ko), ptr(vals), ptr(vo), capacity, ptr(n_dev), 0, bits, ptr(ws), ctypes.c_size_t(nb.value), None)
    finally:
        _unforce()
    torch.cuda.synchronize()
    order = torch.sort(live, stable=True).indices
    assert torch.equal(vo[:n].cpu(), order.to(torch.int32)), entry
    assert torch.equal(ko[:n].cpu(), keys[:n].cpu()[order])


def test_sort_pairs_empty_and_bad_range(cuda):
    k = torch.zeros(8, dtype=torch.int16, device=cuda)
    v = torch.zeros(8, dtype=torch.int32, device=cuda)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=cuda)
    args = lambda n, b, e: (ctypes.c_void_p(k.data_ptr()), ctypes.c_void_p(k.data_ptr()), ctypes.c_void_p(v.data_ptr()),
                            ctypes.c_void_p(v.data_ptr()), n, b, e, ctypes.c_void_p(ws.data_ptr()), ctypes.c_size_t(ws.numel()), None)
    _lib.call("lgs_sort_pairs_u16", *args(0, 0, 14))            # n = 0: no-op
    with pytest.raises(_lib.LiteGSB200Error):
        _lib.call("lgs_sort_pairs_u16", *args(8, 0, 17))
    with pytest.raises(_lib.LiteGSB200Error):
        _lib.call("lgs_sort_pairs_u16", *args(8, 0, 14)[:8] + (ctypes.c_size_t(16), None))
