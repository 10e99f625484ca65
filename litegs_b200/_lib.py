"""ctypes binding of liblitegs_b200.so (the C ABI declared in include/litegs_b200.h).

There is NO fallback: if the library is missing or a call fails, a RuntimeError is raised.  The CPU
oracle under ``oracle/`` is test infrastructure and is never imported from here.
"""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("LITEGS_B200_LIB") or os.path.join(_HERE, "liblitegs_b200.so")   # env: A/B builds only

_P, _I, _D, _Z, _F = ctypes.c_void_p, ctypes.c_int, ctypes.c_double, ctypes.c_size_t, ctypes.c_float

# name -> argument ctypes, in header order (include/litegs_b200.h)
SIGNATURES = {
    "lgs_frustum_culling_aabb": [_P, _P, _P, _I, _I, _P, _P, _P, _P],
    "lgs_cull_compact_activate": [_I, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P],
    "lgs_activate_backward": [_I, _P, _P, _P, _I, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P,
                              _P, _P, _P, _P, _P, _P, _P],
    "lgs_mvp_transform_forward": [_P, _P, _P, _P, _I, _I, _P, _P, _P],
    "lgs_mvp_transform_backward": [_P, _P, _P, _P, _P, _P, _I, _I, _P, _P],
    "lgs_create_transform_matrix_forward": [_P, _P, _P, _I, _P, _P],
    "lgs_create_transform_matrix_backward": [_P, _P, _P, _P, _I, _P, _P, _P],
    "lgs_jacobian_rayspace": [_P, _P, _P, _I, _I, _I, _I, _P, _P],
    "lgs_create_cov2d_forward": [_P, _P, _P, _P, _I, _I, _P, _P],
    "lgs_create_cov2d_backward": [_P, _P, _P, _P, _P, _I, _I, _P, _P],
    "lgs_eigh_and_inv_2x2_forward": [_P, _P, _I, _I, _P, _P, _P, _P],
    "lgs_inv_2x2_backward": [_P, _P, _P, _I, _I, _P, _P],
    "lgs_sh2rgb_forward": [_I, _P, _P, _P, _I, _I, _P, _P],
    "lgs_sh2rgb_backward": [_I, _P, _I, _P, _I, _I, _P, _P, _P, _P],
    "lgs_get_allocate_size": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P],
    "lgs_create_table_workspace_bytes": [_I, _I, ctypes.POINTER(_Z)],
    "lgs_create_table": [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _Z, _P],
    "lgs_set_exact_tile_bound": [_I],
    "lgs_tile_range": [_P, _I, _I, _I, _I, _P, _P],
    "lgs_sort_pairs_u16_workspace_bytes": [_I, ctypes.POINTER(_Z)],
    "lgs_sort_pairs_u16": [_P, _P, _P, _P, _I, _I, _I, _P, _Z, _P],
    "lgs_sort_pairs_u32_workspace_bytes": [_I, ctypes.POINTER(_Z)],
    "lgs_sort_pairs_u32": [_P, _P, _P, _P, _I, _I, _I, _P, _Z, _P],
    "lgs_scan_gathered_workspace_bytes": [_I, ctypes.POINTER(_Z)],
    "lgs_view_params": [_P, _I, _I, _I, _P, _P, _P],
    "lgs_sort_pairs_u32_dev": [_P, _P, _P, _P, _I, _P, _P, _I, _P, _Z, _P],
    "lgs_sort_pairs_u16_dev": [_P, _P, _P, _P, _I, _P, _I, _I, _P, _Z, _P],
    "lgs_sort_pairs_u32k_dev": [_P, _P, _P, _P, _I, _P, _I, _I, _P, _Z, _P],
    "lgs_scan_gathered_dev": [_P, _P, _I, _P, _P, _P, _Z, _P],
    "lgs_emit_pairs_dev": [_P, _P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P],
    "lgs_tile_range_u16_dev": [_P, _I, _P, _I, _I, _P, _P],
    "lgs_tile_range_dev": [_P, _I, _P, _I, _I, _P, _P],
    "lgs_pack_params": [_P, _P, _P, _P, _I, _I, _I, _I, _P, _P],
    "lgs_rasterize_forward_packed": [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P,
                                     _P, _P],
    "lgs_tile_order": [_P, _I, _I, _P, _P],
    "lgs_rasterize_backward": [_P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I,
                               _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P],
    "lgs_set_staging": [_I],
    "lgs_set_sort_impl": [_I],
    "lgs_set_radix_form": [_I],
    "lgs_set_warps_per_block": [_I],
    "lgs_set_backward_reduce": [_I],
    "lgs_set_backward_kernel": [_I],
    "lgs_set_forward_pairs": [_I],
    "lgs_set_err_square_mode": [_I],
    "lgs_set_deterministic": [_I],
    "lgs_project_forward": [_I, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _I, _P,
                            _P],
    "lgs_project_backward": [_I, _P, _P, _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _I,
                             _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _I, _P, _P, _I, _I, _P, _P],
    "lgs_create_viewproj_forward": [_P, _P, _I, _I, _I, _F, _F, _P, _P, _P, _P, _P],
    "lgs_create_viewproj_backward": [_P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _P, _P, _P],
    "lgs_adam_update_chunk": [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _D, _D, _D, _D, _P],
    "lgs_adam_update_primitive": [_P, _P, _P, _P, _P, _I, _I, _D, _D, _D, _D, _P],
    "lgs_sparse_chunk_op": [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P],
    "lgs_mark_visible_chunks": [_P, _P, _I, _P, _P],
    "lgs_nvls_allreduce_f32": [_P, _Z, _I, _I, _I, _P],
    "lgs_morton_codes": [_P, _P, _P, _I, _I, _P, _P],
    "lgs_permute_rows": [_P, _P, _I, _I, _P, _P],
    "lgs_cluster_aabb": [_P, _P, _P, _I, _I, _P, _P, _P],
    "lgs_filter_3d": [_P, _I, _I, _P, _P, _P, _I, _P, _P],
    "lgs_adam_step_dense": [_P, _P, _P, _P, _P, _P, _P, _I, _I, _D, _D, _D, _I, _P],
    "lgs_ssim_num_block_sums": [_I, _I, _I, _I, ctypes.POINTER(_I)],
    "lgs_ssim_forward": [_P, _P, _I, _I, _I, _I, _F, _F, _I, _F, _P, _P, _P, _P, _P, _P],
    "lgs_ssim_backward": [_P, _P, _P, _F, _P, _P, _P, _I, _I, _I, _I, _I, _F, _P, _P],
    "lgs_depth_normal_num_block_sums": [_I, _I, ctypes.POINTER(_I)],
    "lgs_depth_normal": [_P, _I, _P, _I, _P, _I, _I, _P, _I, _I, _F, _F, _P, _P, _P, _P, _P, _P],
    "lgs_tsdf_integrate": [_P, _P, _P, _I, _I, _I, _F, _F, _F, _F, _F, _P, _P, _P, _P, _P, _I, _I, _I, _F, _F, _P],
    "lgs_mesh_count": [_P, _P, _I, _I, _I, _F, _P, _P, _P, _P],
    "lgs_mesh_emit": [_P, _P, _I, _I, _I, _F, _F, _F, _F, _P, _P, _P, _P, ctypes.c_longlong, ctypes.c_longlong, _P, _P, _P, _P],
}
NO_STATUS = {"lgs_last_error": ctypes.c_char_p, "lgs_abi_version": ctypes.c_int}

_lib = None


class LiteGSB200Error(RuntimeError):
    pass


def load() -> ctypes.CDLL:
    """Load the shared library and attach prototypes.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise LiteGSB200Error(
            f"{LIB_PATH} not found: build it with `python -m litegs_b200.build` (nvcc, sm_90a). "
            "litegs_b200 has no CPU or PyTorch fallback.")
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = ctypes.c_int
    for name, restype in NO_STATUS.items():
        fn = getattr(lib, name)
        fn.argtypes = []
        fn.restype = restype
    _lib = lib
    return lib


def exported_symbols():
    """Every symbol the header declares (used by the CPU-side ABI test)."""
    return list(SIGNATURES) + list(NO_STATUS)


def call(name: str, *args) -> None:
    """Invoke a status-returning entry point; raise with the library's message on failure."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.lgs_last_error()
        raise LiteGSB200Error(f"{name} failed (code {rc}): {msg.decode() if msg else ''}")
