"""Cost of the device-side count entry points on the C2 sizes: the tile sort of D = 10.9 M (u16 key, i32 value) pairs on 14 bits
against its host-count form, the depth sort of 1 M u32 keys on 24 bits and the gathered scan of 1 M (these two have the
device-count form only); and the host-count tile sort at the C4 size."""
import ctypes
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
import torch
from litegs_b200 import _lib

dev = torch.device("cuda:0")
st = lambda: torch.cuda.current_stream().cuda_stream
P = lambda t: t.data_ptr()


def timeit(fn, n=30):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1000.0


D = 10_897_674
for cap in (D, int(D * 1.3) + 65536):
    keys = torch.randint(1, 16201, (cap,), device=dev, dtype=torch.int32).to(torch.int16)
    vals = torch.arange(cap, device=dev, dtype=torch.int32)
    ko, vo = torch.empty_like(keys), torch.empty_like(vals)
    nb = ctypes.c_size_t(0)
    _lib.call("lgs_sort_pairs_u16_workspace_bytes", cap, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    ndev = torch.tensor([D], dtype=torch.int32, device=dev)
    t_host = timeit(lambda: _lib.call("lgs_sort_pairs_u16", P(keys), P(ko), P(vals), P(vo), D, 0, 14, P(ws), ctypes.c_size_t(nb.value), st()))
    t_dev = timeit(lambda: _lib.call("lgs_sort_pairs_u16_dev", P(keys), P(ko), P(vals), P(vo), cap, P(ndev), 0, 14, P(ws), ctypes.c_size_t(nb.value), st()))
    print(f"tile sort D={D} capacity={cap}: host count {t_host:.1f} us, device count {t_dev:.1f} us")

N = 1_000_064
k32 = torch.randint(0, 1 << 24, (N,), device=dev, dtype=torch.int32)
v32 = torch.arange(N, device=dev, dtype=torch.int32)
ko, vo = torch.empty_like(k32), torch.empty_like(v32)
nb = ctypes.c_size_t(0)
_lib.call("lgs_sort_pairs_u32_workspace_bytes", N, ctypes.byref(nb))
ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
ndev = torch.tensor([984_960], dtype=torch.int32, device=dev)
bias = torch.zeros(1, dtype=torch.int32, device=dev)
t_dev = timeit(lambda: _lib.call("lgs_sort_pairs_u32_dev", P(k32), P(ko), P(v32), P(vo), N, P(ndev), P(bias), 24, P(ws), ctypes.c_size_t(nb.value), st()))
print(f"depth sort N=984960 (capacity {N}): device count {t_dev:.1f} us")
cnt = torch.randint(0, 20, (N,), device=dev, dtype=torch.int32)
out = torch.empty(N, dtype=torch.int32, device=dev)
nb2 = ctypes.c_size_t(0)
_lib.call("lgs_scan_gathered_workspace_bytes", N, ctypes.byref(nb2))
ws2 = torch.empty(nb2.value, dtype=torch.uint8, device=dev)
order = torch.randperm(N, device=dev).to(torch.int32)
t_dev = timeit(lambda: _lib.call("lgs_scan_gathered_dev", P(cnt), P(order), N, P(ndev), P(out), P(ws2), ctypes.c_size_t(nb2.value), st()))
print(f"gathered scan: device count {t_dev:.1f} us")

# C4-sized tile sort (71.7 M pairs, 16 bits)
D4 = 71_700_532
keys = torch.randint(1, 64801, (D4,), device=dev, dtype=torch.int32).to(torch.int16)
vals = torch.arange(D4, device=dev, dtype=torch.int32)
ko, vo = torch.empty_like(keys), torch.empty_like(vals)
nb = ctypes.c_size_t(0)
_lib.call("lgs_sort_pairs_u16_workspace_bytes", D4, ctypes.byref(nb))
ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
t = timeit(lambda: _lib.call("lgs_sort_pairs_u16", P(keys), P(ko), P(vals), P(vo), D4, 0, 16, P(ws), ctypes.c_size_t(nb.value), st()), n=10)
print(f"C4 tile sort D={D4}, 16 bits, LGS_RS_IPT={os.environ.get('LGS_RS_IPT', 'default')}, LGS_SORT={os.environ.get('LGS_SORT', 'lgs')}: {t:.1f} us "
      f"= {D4 * (2 + 2 * 12) / t / 1e6:.2f} TB/s of algorithmic traffic")
