"""Generates the CPU-side fixtures that pin this project to facts of the reference source tree (LiteGS), so that the tests
that check them run without it:

    python tests/golden/make_golden_reference_cpu.py /path/to/LiteGS      # writes into tests/golden/

reference_abi.json           -- the 26 pybind names of gaussian_raster/ext_cuda.cpp and each one's declared argument count
                                (raster.h, binning.h, compact.h, transform.h); read by tests/test_abi.py.
reference_line_counts.json   -- the number of lines of every .cu/.cuh/.h/.py/.cpp file under litegs/; read by
                                tests/test_citations.py to resolve `<file>:<line>` citations.
colmap_reference_read.npz    -- what the reference's COLMAP reader (litegs/io_manager/colmap.py, its two heavy imports
                                stubbed) returns for the model tests/test_colmap.py writes, plus the SHA-256 of the three
                                files it read; read by tests/test_colmap.py.
"""
import hashlib
import importlib.util
import json
import os
import re
import sys
import tempfile
import types

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
HERE = os.path.dirname(os.path.abspath(__file__))
COLMAP_FILES = ("cameras.bin", "images.bin", "points3D.bin")


def reference_abi(ref):
    gr = os.path.join(ref, "litegs", "submodules", "gaussian_raster")
    names = re.findall(r'm\.def\("(\w+)"', open(os.path.join(gr, "ext_cuda.cpp")).read())
    decl = "".join(open(os.path.join(gr, h)).read() for h in ("raster.h", "binning.h", "compact.h", "transform.h"))
    decl = re.sub(r"//.*", "", decl)
    out = {}
    for name in names:
        m = re.search(r"\b" + name + r"\s*\(([^;]*?)\)\s*;", decl, flags=re.S)
        out[name] = len([a for a in m.group(1).split(",") if a.strip()])
    return out


def line_counts(ref):
    out = {}
    for d, dirs, files in os.walk(os.path.join(ref, "litegs")):
        dirs[:] = sorted(x for x in dirs if x != "__pycache__")
        for f in sorted(files):
            if f.endswith((".cu", ".cuh", ".h", ".py", ".cpp")):
                p = os.path.join(d, f)
                out[os.path.relpath(p, ref)] = sum(1 for _ in open(p, errors="replace"))
    return out


def reference_reader(ref):
    """litegs/io_manager/colmap.py imported on its own: `plyfile` and `litegs.data` (pulls in cv2/torch datasets) are
    replaced by stubs that record the constructor arguments."""
    pkg_dir = os.path.join(ref, "litegs")
    path = os.path.join(pkg_dir, "io_manager", "colmap.py")
    saved = {k: sys.modules.get(k) for k in ("plyfile", "litegs", "litegs.data", "litegs.io_manager", "litegs.io_manager.colmap")}
    try:
        ply = types.ModuleType("plyfile"); ply.PlyData = object; ply.PlyElement = object
        pkg = types.ModuleType("litegs"); pkg.__path__ = [pkg_dir]
        iom = types.ModuleType("litegs.io_manager"); iom.__path__ = [os.path.join(pkg_dir, "io_manager")]
        data = types.ModuleType("litegs.data")

        class PinHoleCameraInfo:
            def __init__(self, id, width, height, parameters):
                self.id, self.width, self.height, self.parameters = id, width, height, np.array(parameters)

        class ImageFrame:
            def __init__(self, id, qvec, tvec, camera_id, name, img_source, xys):
                self.id, self.qvec, self.tvec, self.camera_id, self.name, self.img_source, self.xys = id, qvec, tvec, camera_id, name, img_source, xys

        data.PinHoleCameraInfo, data.ImageFrame, data.CameraInfo = PinHoleCameraInfo, ImageFrame, object
        sys.modules.update({"plyfile": ply, "litegs": pkg, "litegs.io_manager": iom, "litegs.data": data})
        spec = importlib.util.spec_from_file_location("litegs.io_manager.colmap", path)
        mod = importlib.util.module_from_spec(spec)
        sys.modules["litegs.io_manager.colmap"] = mod
        spec.loader.exec_module(mod)
        return mod
    finally:
        for k, v in saved.items():
            if v is None:
                sys.modules.pop(k, None)
            else:
                sys.modules[k] = v


def colmap_read(ref):
    from litegs_b200 import colmap
    from tests.test_colmap import READER_MODEL, _model
    rd = reference_reader(ref)
    with tempfile.TemporaryDirectory() as d:
        colmap.write_model(d, *_model(**READER_MODEL))
        sparse = os.path.join(d, "sparse", "0")
        out = {f"sha256_{f}": np.array(hashlib.sha256(open(os.path.join(sparse, f), "rb").read()).hexdigest()) for f in COLMAP_FILES}
        cam_dict, frames = rd.load_frames(d, "images")
        out["camera_ids"] = np.array(sorted(cam_dict))
        for k, c in cam_dict.items():
            out[f"camera_{k}_size"] = np.array([c.width, c.height])
            out[f"camera_{k}_params"] = np.asarray(c.parameters)
        out["frame_names"] = np.array([f.name for f in frames])
        out["frame_ids"] = np.array([f.id for f in frames])
        out["frame_camera_ids"] = np.array([f.camera_id for f in frames])
        out["frame_qvec"] = np.stack([np.asarray(f.qvec) for f in frames])
        out["frame_tvec"] = np.stack([np.asarray(f.tvec) for f in frames])
        for i, f in enumerate(frames):
            out[f"frame_{i}_xys"] = np.asarray(f.xys).reshape(-1, 2)
        xyz, rgb, err = rd.__dict__["__read_points3D_binary"](os.path.join(sparse, "points3D.bin"))
        out["points_xyz"], out["points_rgb"], out["points_err"] = np.asarray(xyz), np.asarray(rgb), np.asarray(err)
    return out


def main():
    ref = sys.argv[1]
    json.dump(reference_abi(ref), open(os.path.join(HERE, "reference_abi.json"), "w"), indent=1, sort_keys=True)
    json.dump(line_counts(ref), open(os.path.join(HERE, "reference_line_counts.json"), "w"), indent=1, sort_keys=True)
    np.savez_compressed(os.path.join(HERE, "colmap_reference_read.npz"), **colmap_read(ref))


if __name__ == "__main__":
    main()
