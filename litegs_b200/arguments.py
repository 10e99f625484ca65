"""Hot-path-relevant pipeline parameters (defaults of the reference's ``PipelineParams``,
litegs/arguments.py:69-77).  Any object with these attributes is accepted by ``litegs_b200.render``."""
from dataclasses import dataclass


@dataclass
class PipelineParams:
    cluster_size: int = 128
    tile_size: tuple = (8, 16)
    sparse_grad: bool = True
    enable_transmitance: bool = False
    enable_depth: bool = False
    input_color_type: str = "sh"
    # ours, not the reference's: antialiased mode of the fused path (DESIGN.md section 1).  Readers use
    # getattr(pp, "antialiased", False), so the reference's own PipelineParams keeps working.
    antialiased: bool = False
    # ours as well: exact gradient mode of the fused path's backward (DESIGN.md section 1), read as getattr(pp, "exact_grad", False)
    exact_grad: bool = False
    # ours as well: per-pixel depth on the fused path (DESIGN.md section 1, "Depth"), read as getattr(pp, "render_depth", False);
    # enable_depth above keeps the reference's meaning
    render_depth: bool = False
    # ours as well: per-pixel normals on the fused path (DESIGN.md section 1, "Normals"), read as getattr(pp, "render_normal", False)
    render_normal: bool = False
