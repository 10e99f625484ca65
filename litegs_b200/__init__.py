"""litegs_b200 -- an H100-native (sm_90a) differentiable 3D Gaussian Splatting render path behind MooreThreads/LiteGS's
operator surface.

    fused       the 26 entry points of the reference's ``litegs_fused`` pybind module, on the C ABI (include/litegs_b200.h)
    wrapper     the reference's autograd operators (``litegs/utils/wrapper.py`` names and signatures)
    render      render_preprocess / render (reference surface), render_view (fused), render_views (multi-view, streams)
    pipeline    the fused per-view forward / backward
    ssim        the reference's ``fused_ssim`` package surface + l1_ssim_loss_and_grad
    optimizer   FusedAdam (the reference's sparse Adam in one launch), its learning-rate schedule
    dist        view sharding, dense gradient accumulator, all-reduce
    scene       synthetic scenes / cameras / chunking used by tests and the bench

Nothing here runs on the CPU: the CUDA library (``python -m litegs_b200.build``) is required and its absence raises.
"""
__version__ = "0.1.0"
